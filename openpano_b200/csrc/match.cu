// match.cu — exact pairwise descriptor matching.
//
// Replaces PairWiseMatcher::match (feature/matcher.cc:90-135) with the exact rule
// of FeatureMatcher::match (feature/matcher.cc:15-71), the parity contract
// (SURVEY.md §8c).  Distances are feature/dist.cc:22-57's SSE branch bit for bit:
// four lane accumulators over the 32 4-float steps, summed (l0+l1)+(l2+l3), no
// FMA.  The reference's rule
//     loop k over the smaller set: exact top-2 of row k (lowest index wins);
//     reject if min > R*next; next = min(next, min_{kk!=k} d(best, kk)); reject again
// is evaluated from two symmetric top-2 reductions (rows of A over B, rows of B
// over A): min_{kk!=k} d(j, kk) is column j's second minimum when its argmin is
// k, and its minimum otherwise.
//
// Two ways to get those reductions:
//  * tensor path (default): match_tc.cu nominates (approx best, argmin, approx
//    second) per row on the tensor cores (wgmma); here every row gets its exact
//    fp32 best distance, a certified interval for its second-best (the fp16
//    quantisation bound), and rows whose argmin or accept/reject decision is not
//    certain within those intervals are re-scanned exactly (k_exact_rows).  The
//    outcome is the reference's, bit for bit; the tensor cores only decide how
//    little exact work is left.
//    COLUMNS ON DEMAND (large runs): the reference only walks column j (matcher.cc:57-61)
//    for rows that passed their own ratio test, so the second reduction is needed for
//    few rows of the larger set.  With enough work to fill the GPU anyway, only the
//    smaller set's rows go through the first tensor pass; the rows of the larger set
//    start UNKNOWN and the decide rounds request exactly the columns they need, which a
//    gathered top-2 tensor pass then nominates (PANO_MATCH_LAZY=0/1 forces either way).
//  * exact path (PANO_MATCH_PATH=exact): both reductions in fp32 on the CUDA
//    cores (k_match_top2), kept as the in-engine cross-check.
#include "sift.cuh"
#include "match_tc.cuh"
#include <float.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>

// feature/dist.cc:22-57 (SSE lane order); a and b are 16-byte aligned rows of 128 floats
__device__ __forceinline__ float exact_dist(const float* __restrict__ a, const float* __restrict__ b) {
  float l0 = 0.f, l1 = 0.f, l2 = 0.f, l3 = 0.f;
  const float4* pa = (const float4*)a;
  const float4* pb = (const float4*)b;
#pragma unroll 8
  for (int k = 0; k < 32; ++k) {
    float4 x = __ldg(pa + k), y = __ldg(pb + k);
    float d0 = x.x - y.x, d1 = x.y - y.y, d2 = x.z - y.z, d3 = x.w - y.w;
    l0 += d0 * d0; l1 += d1 * d1; l2 += d2 * d2; l3 += d3 * d3;
  }
  return (l0 + l1) + (l2 + l3);
}

__device__ __forceinline__ void top2_merge(float& mn, int& idx, float& sec, float m2, int i2, float s2) {
  if (m2 < mn || (m2 == mn && i2 < idx)) { sec = fminf(mn, s2); mn = m2; idx = i2; }
  else sec = fminf(sec, m2);
}

// ============================================================ exact path (fp32 CUDA cores)
#define MT 64            // rows of the query tile and of the target tile
#define MT_STRIDE 132    // padded row stride in floats (conflict-free float4 reads)
#define MT_THREADS 256

struct MatchTask {       // one top-2 reduction: rows [q_row0, q_row0+MT) of Q against all of T
  long long q_base, t_base;  // first descriptor row of the sets inside the featureset
  int q_n, t_n;
  int q_row0;
  long long res_off;     // where this query set's results start
};

// Per-row knowledge, as certified intervals.  state bit 1: argmin certain (then
// mn == mn_hi is the exact fp32 distance to idx); bit 0: second-best exact
// (sec_lo == sec_hi).  With an uncertain argmin only the bounds are valid.  Bit 2: nothing is
// known yet (columns on demand: the row has not been through a tensor pass).
struct RowInfo { float mn, mn_hi; int idx; float sec_lo, sec_hi; int state; int requested; int pad; };

__global__ void __launch_bounds__(MT_THREADS)
k_match_top2(const float* __restrict__ desc, const MatchTask* __restrict__ tasks, RowInfo* __restrict__ res) {
  extern __shared__ float sm[];
  float* sq = sm;                       // [MT][MT_STRIDE]
  float* st = sm + MT * MT_STRIDE;      // [MT][MT_STRIDE]
  const MatchTask tk = tasks[blockIdx.x];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const float* Q = desc + tk.q_base * 128;
  const float* T = desc + tk.t_base * 128;

  for (int i = tid; i < MT * 32; i += MT_THREADS) {   // 32 float4 per row
    int r = i >> 5, c4 = i & 31;
    int gr = tk.q_row0 + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (gr < tk.q_n) v = __ldg((const float4*)(Q + (size_t)gr * 128) + c4);
    *(float4*)(sq + r * MT_STRIDE + c4 * 4) = v;
  }

  float bmn[4], bsec[4];
  int bidx[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { bmn[i] = FLT_MAX; bsec[i] = FLT_MAX; bidx[i] = 0x7fffffff; }

  for (int t0 = 0; t0 < tk.t_n; t0 += MT) {
    __syncthreads();
    for (int i = tid; i < MT * 32; i += MT_THREADS) {
      int r = i >> 5, c4 = i & 31;
      int gr = t0 + r;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gr < tk.t_n) v = __ldg((const float4*)(T + (size_t)gr * 128) + c4);
      *(float4*)(st + r * MT_STRIDE + c4 * 4) = v;
    }
    __syncthreads();
    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int l = 0; l < 4; ++l) acc[i][j][l] = 0.f;
#pragma unroll 4
    for (int k = 0; k < 32; ++k) {
      float4 a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = *(const float4*)(sq + (ty + 16 * i) * MT_STRIDE + k * 4);
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = *(const float4*)(st + (tx + 16 * j) * MT_STRIDE + k * 4);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float d0 = a[i].x - b[j].x, d1 = a[i].y - b[j].y, d2 = a[i].z - b[j].z, d3 = a[i].w - b[j].w;
          acc[i][j][0] += d0 * d0; acc[i][j][1] += d1 * d1;
          acc[i][j][2] += d2 * d2; acc[i][j][3] += d3 * d3;
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int col = t0 + tx + 16 * j;
        if (col < tk.t_n) {
          float d = (acc[i][j][0] + acc[i][j][1]) + (acc[i][j][2] + acc[i][j][3]);
          // ascending col within a thread: strict < keeps the lowest index
          if (d < bmn[i]) { bsec[i] = bmn[i]; bmn[i] = d; bidx[i] = col; }
          else if (d < bsec[i]) bsec[i] = d;
        }
      }
  }
  // merge the 16 threads (tx) that share a query row: they sit in one half-warp
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float mn = bmn[i], sec = bsec[i];
    int idx = bidx[i];
#pragma unroll
    for (int off = 8; off >= 1; off >>= 1) {
      float m2 = __shfl_xor_sync(0xffffffffu, mn, off);
      float s2 = __shfl_xor_sync(0xffffffffu, sec, off);
      int i2 = __shfl_xor_sync(0xffffffffu, idx, off);
      top2_merge(mn, idx, sec, m2, i2, s2);
    }
    int row = tk.q_row0 + ty + 16 * i;
    if (tx == 0 && row < tk.q_n) {
      RowInfo o; o.mn = mn; o.mn_hi = mn; o.idx = idx; o.sec_lo = sec; o.sec_hi = sec; o.state = 3; o.requested = 0; o.pad = 0;
      res[tk.res_off + row] = o;
    }
  }
}

// ============================================================ tensor path: certification

struct SideMeta {        // one query set of one pair
  long long q_base, t_base;   // descriptor rows in the featureset
  int q_n, t_n;
  long long res_off;          // RowInfo / TcTop2 offset of this side
  int r0, r1;                 // rows of this side that went through the first pass (a row-sharded call
                              // nominates only its own rows of the smaller set; otherwise 0 .. q_n)
  int parts, pad;             // first pass split into `parts` column ranges (tail balance); part p's
                              // nominations sit at approx[p * res_total + res_off + row]
};

// Bound on |approx d^2 - exact fp32 d^2| for a query of squared norm nq against
// targets of squared norm <= nmax: fp16 rounding of both operands (2 * 2^-11
// relative on every product, doubled by the -2ab term) plus the packed-key
// mantissa truncation, the hi/lo norm split and accumulation slack.
__device__ __forceinline__ float tc_eps(float nq, float nmax) {
  return 0.00215f * sqrtf(nq * nmax) + 0.0005f * nmax + 1.0f;
}

__device__ __forceinline__ RowInfo refine_row(const float* __restrict__ desc, const SideMeta& sm, int r, const TcTop2 ap,
                                              float eps, float ratio_sqr) {
  RowInfo o;
  o.requested = 0; o.pad = 0;
  const bool idx_ok = ap.idx >= 0 && ap.idx < sm.t_n;
  o.idx = idx_ok ? ap.idx : 0;
  const bool single = ap.m2 == FLT_MAX;                 // only one real target
  const bool certain = idx_ok && (single || (ap.m2 - ap.m1 > 2.f * eps));
  if (sm.t_n <= 0) { o.mn = FLT_MAX; o.mn_hi = FLT_MAX; o.sec_lo = FLT_MAX; o.sec_hi = FLT_MAX; o.state = 3; }
  else if (certain && !single && (ap.m1 - eps) > ratio_sqr * (ap.m2 + eps)) {
    // The argmin is certain and so is the outcome of the row's ratio test (min > R * next_min for every
    // distance inside the error band): the row is rejected whatever its exact distance is, so the 1 KB
    // exact re-computation is skipped and the row keeps certified BOUNDS.  k_match_decide rejects it
    // at its first test (mn_lo > R * min(sec_hi, .)); as a column of another row it still offers
    // valid bounds [mn, mn_hi] / [sec_lo, sec_hi] — in an all-pairs run nearly every row of a
    // non-overlapping image pair ends here.
    o.mn = ap.m1 - eps; o.mn_hi = ap.m1 + eps;
    o.sec_lo = fmaxf(ap.m2 - eps, o.mn); o.sec_hi = ap.m2 + eps;
    o.state = 2;
  }
  else if (certain) {
    // the argmin is certain: its exact fp32 distance is the row minimum
    o.mn = exact_dist(desc + (size_t)(sm.q_base + r) * 128, desc + (size_t)(sm.t_base + o.idx) * 128);
    o.mn_hi = o.mn;
    if (single) { o.sec_lo = FLT_MAX; o.sec_hi = FLT_MAX; o.state = 3; }
    else { o.sec_lo = fmaxf(ap.m2 - eps, o.mn); o.sec_hi = fmaxf(ap.m2 + eps, o.mn); o.state = 2; }
  } else {
    // two or more targets within the error band of the best: only bounds are known
    o.mn = fmaxf(ap.m1 - eps, 0.f); o.mn_hi = ap.m1 + eps;
    o.sec_lo = fmaxf(ap.m2 - eps, 0.f); o.sec_hi = ap.m2 + eps;
    o.state = 0;
  }
  return o;
}

// lazy != 0: the sides of the larger sets (odd side indices) have not been through the tensor
// pass; their rows start unknown and are nominated on request (k_refine_gathered).
__device__ __forceinline__ void refine_side_row(const float* __restrict__ desc, const float* __restrict__ norms,
                                                const unsigned* __restrict__ maxnorm_bits, const SideMeta* __restrict__ sides,
                                                TcTop2* __restrict__ approx, long long res_total, float ratio_sqr, int lazy,
                                                RowInfo* __restrict__ info, int side, int r) {
  const SideMeta sm = sides[side];
  if (r >= sm.q_n) return;
  if (r < sm.r0 || r >= sm.r1) return;      // another shard's row: never decided, never a column here
  if (lazy && (side & 1) && sm.t_n > 0) {
    RowInfo o; o.mn = 0.f; o.mn_hi = FLT_MAX; o.idx = 0; o.sec_lo = 0.f; o.sec_hi = FLT_MAX; o.state = 4; o.requested = 0; o.pad = 0;
    info[sm.res_off + r] = o;
    return;
  }
  const float nmax = __uint_as_float(*maxnorm_bits);
  TcTop2 ap = approx[sm.res_off + r];
  if (sm.parts > 1) {
    // the column ranges ascend with the part index, so on equal scores the earlier part keeps the
    // argmin: the same "lowest column" rule as inside one part
    for (int p = 1; p < sm.parts; ++p) {
      const TcTop2 q = approx[(long long)p * res_total + sm.res_off + r];
      if (q.m1 < ap.m1) { ap.m2 = fminf(ap.m1, q.m2); ap.m1 = q.m1; ap.idx = q.idx; }
      else ap.m2 = fminf(ap.m2, q.m1);
    }
    approx[sm.res_off + r] = ap;     // where the filter pass looks for the row's threshold
  }
  info[sm.res_off + r] = refine_row(desc, sm, r, ap, tc_eps(norms[sm.q_base + r], nmax), ratio_sqr);
}

// sides on gridDim.y, which stops at 65,535: the blocks of a y index take every gridDim.y-th side
__global__ void k_refine(const float* __restrict__ desc, const float* __restrict__ norms,
                         const unsigned* __restrict__ maxnorm_bits, const SideMeta* __restrict__ sides, int n_sides,
                         TcTop2* __restrict__ approx, long long res_total, float ratio_sqr, int lazy,
                         RowInfo* __restrict__ info) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  for (int side = blockIdx.y; side < n_sides; side += gridDim.y)
    refine_side_row(desc, norms, maxnorm_bits, sides, approx, res_total, ratio_sqr, lazy, info, side, r);
}

// The same certification for rows nominated on request: gathered row g carries (side, row) in
// g_meta and its nomination in g_approx[g]; the nomination is also stored at the row's own slot,
// where a later filter pass looks for its threshold.
__global__ void k_refine_gathered(const float* __restrict__ desc, const float* __restrict__ norms,
                                  const unsigned* __restrict__ maxnorm_bits, const SideMeta* __restrict__ sides,
                                  const int2* __restrict__ g_meta, const TcTop2* __restrict__ g_approx,
                                  const int* __restrict__ n_blocks, float ratio_sqr, TcTop2* __restrict__ approx,
                                  RowInfo* __restrict__ info) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= *n_blocks * 128) return;
  const int2 me = g_meta[g];
  if (me.x < 0) return;
  const SideMeta sm = sides[me.x];
  const TcTop2 ap = g_approx[g];
  const float nmax = __uint_as_float(*maxnorm_bits);
  approx[sm.res_off + me.y] = ap;
  info[sm.res_off + me.y] = refine_row(desc, sm, me.y, ap, tc_eps(norms[sm.q_base + me.y], nmax), ratio_sqr);
}

// Exact re-scan of listed rows: one 256-thread block per row, every thread strides
// over the targets (the list is short, so parallelism has to come from the row).
__global__ void __launch_bounds__(256)
k_exact_rows(const float* __restrict__ desc, const SideMeta* __restrict__ sides, const int2* __restrict__ list,
             const int* __restrict__ list_count, RowInfo* __restrict__ info) {
  __shared__ __align__(16) float sq[128];
  __shared__ float s_mn[8], s_sec[8];
  __shared__ int s_idx[8];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int n = *list_count;
  for (int e = blockIdx.x; e < n; e += gridDim.x) {
    const int2 it = list[e];
    const SideMeta sm = sides[it.x];
    const float* q = desc + (size_t)(sm.q_base + it.y) * 128;
    __syncthreads();
    if (tid < 32) *(float4*)(&sq[tid * 4]) = __ldg((const float4*)q + tid);
    __syncthreads();
    float mn = FLT_MAX, sec = FLT_MAX;
    int idx = 0x7fffffff;
    for (int c = tid; c < sm.t_n; c += 256) {
      const float4* pb = (const float4*)(desc + (size_t)(sm.t_base + c) * 128);
      // the whole 512-byte target row is requested before any arithmetic: the kernel
      // is load-latency bound, so all 32 loads of a row must be in flight together
      float4 yv[32];
#pragma unroll
      for (int k = 0; k < 32; ++k) yv[k] = __ldg(pb + k);
      float l0 = 0.f, l1 = 0.f, l2 = 0.f, l3 = 0.f;
#pragma unroll
      for (int k = 0; k < 32; ++k) {
        const float4 x = *(const float4*)(&sq[k * 4]), y = yv[k];
        float d0 = x.x - y.x, d1 = x.y - y.y, d2 = x.z - y.z, d3 = x.w - y.w;
        l0 += d0 * d0; l1 += d1 * d1; l2 += d2 * d2; l3 += d3 * d3;
      }
      float d = (l0 + l1) + (l2 + l3);
      if (d < mn) { sec = mn; mn = d; idx = c; }
      else if (d < sec) sec = d;
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
      float m2 = __shfl_xor_sync(0xffffffffu, mn, off);
      float s2 = __shfl_xor_sync(0xffffffffu, sec, off);
      int i2 = __shfl_xor_sync(0xffffffffu, idx, off);
      top2_merge(mn, idx, sec, m2, i2, s2);
    }
    if (lane == 0) { s_mn[wid] = mn; s_sec[wid] = sec; s_idx[wid] = idx; }
    __syncthreads();
    if (tid == 0) {
      for (int wdx = 1; wdx < 8; ++wdx) top2_merge(mn, idx, sec, s_mn[wdx], s_idx[wdx], s_sec[wdx]);
      RowInfo o; o.mn = mn; o.mn_hi = mn; o.idx = idx; o.sec_lo = sec; o.sec_hi = sec; o.state = 3; o.requested = 1; o.pad = 0;
      info[sm.res_off + it.y] = o;
    }
  }
}

struct PairMeta {
  int side_small, side_large;    // indices into the side table (small set queries / large set queries)
  int n_small, n_large;
  long long out_off;             // per-row decision of the smaller set
  int rev, pad;                  // the pair was swapped (its first image is the larger set): MatchData::reverse
  int k0, k1;                    // rows of the smaller set this call decides (row-sharded calls; else 0 .. n_small)
};

#define OUT_PENDING (-2)

// Decision per row k of the smaller set (matcher.cc:49-66) from certified
// intervals; rows that cannot be decided request exact re-scans and stay pending.
// Requests go to per-side lists (list_rows[side.res_off + slot], side_cnt[side]) so
// that the gathered second tensor pass can batch the rows of one side together.
// Unknown rows (columns on demand) go to the second list of the side: they need a nomination
// first, not a filter pass.  side_cnt holds [list][side] for this round.
__device__ __forceinline__ void request_row(const SideMeta* __restrict__ sides, RowInfo* __restrict__ info, int side,
                                            int row, int* list_rows, int* list_unknown,
                                            int* __restrict__ side_cnt, int n_sides) {
  const long long off = sides[side].res_off;
  RowInfo* ri = &info[off + row];
  if (atomicExch(&ri->requested, 1) == 0) {
    if (ri->state & 4) list_unknown[off + atomicAdd(&side_cnt[n_sides + side], 1)] = row;
    else list_rows[off + atomicAdd(&side_cnt[side], 1)] = row;
  }
}

__device__ __forceinline__ void match_decide_row(const PairMeta* __restrict__ pairs, const SideMeta* __restrict__ sides,
                                                 RowInfo* __restrict__ info, float ratio_sqr, int first_round,
                                                 int* __restrict__ out, int* __restrict__ total,
                                                 int* list_rows, int* list_unknown, int* __restrict__ side_cnt,
                                                 int n_sides, int pair, int row) {
  const PairMeta pm = pairs[pair];
  const int k = pm.k0 + row;
  if (k >= pm.k1) return;
  const size_t oslot = pm.out_off + k;
  if (!first_round && out[oslot] != OUT_PENDING) return;
  int result = -1;
  if (pm.n_large > 0) {
    const SideMeta ss = sides[pm.side_small], sl = sides[pm.side_large];
    const RowInfo r = info[ss.res_off + k];
    if (!(r.state & 2)) {
      // argmin not certain: the row test alone (mn > R * second) may already reject
      if (r.mn > ratio_sqr * r.sec_hi) result = -1;
      else {
        result = OUT_PENDING;
        request_row(sides, info, pm.side_small, k, list_rows, list_unknown, side_cnt, n_sides);
        // columns on demand: the nominated column is most likely the one this row will need
        if (info[sl.res_off + r.idx].state & 4)
          request_row(sides, info, pm.side_large, r.idx, list_rows, list_unknown, side_cnt, n_sides);
      }
    } else {
      const RowInfo c = info[sl.res_off + r.idx];
      if (c.state & 4) {
        // nothing is known about column r.idx yet: only the row's own test can reject, and only
        // min == 0 accepts whatever the column holds (0 > R * next_min is false for every next_min)
        if (r.mn > ratio_sqr * r.sec_hi) result = -1;
        else if (!(r.mn > 0.f)) result = r.idx;
        else {
          result = OUT_PENDING;
          request_row(sides, info, pm.side_large, r.idx, list_rows, list_unknown, side_cnt, n_sides);
        }
      } else {
        float c_lo, c_hi;
        bool need_c = false;
        if (c.state & 2) {                                  // column's argmin certain
          const bool mine = c.idx == k;
          c_lo = mine ? c.sec_lo : c.mn; c_hi = mine ? c.sec_hi : c.mn_hi;
          need_c = mine && !(c.state & 1);
        } else {                                            // min_{kk != k} d(j, kk) lies between its best and second bounds
          c_lo = c.mn; c_hi = c.sec_hi;
          need_c = true;
        }
        const float nlo = fminf(r.sec_lo, c_lo), nhi = fminf(r.sec_hi, c_hi);
        if (r.mn > ratio_sqr * nhi) result = -1;               // rejected for every admissible next_min
        else if (!(r.mn > ratio_sqr * nlo)) result = r.idx;    // accepted for every admissible next_min
        else {
          result = OUT_PENDING;
          if (!(r.state & 1)) request_row(sides, info, pm.side_small, k, list_rows, list_unknown, side_cnt, n_sides);
          if (need_c) request_row(sides, info, pm.side_large, r.idx, list_rows, list_unknown, side_cnt, n_sides);
        }
      }
    }
  }
  out[oslot] = result;
  if (result >= 0) atomicAdd(total, 1);
}

// pairs on gridDim.y, which stops at 65,535: the blocks of a y index take every gridDim.y-th pair
__global__ void k_match_decide(const PairMeta* __restrict__ pairs, int n_pairs, const SideMeta* __restrict__ sides,
                               RowInfo* __restrict__ info, float ratio_sqr, int first_round,
                               int* __restrict__ out, int* __restrict__ total,
                               int* list_rows, int* list_unknown, int* __restrict__ side_cnt,
                               int n_sides) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  for (int pair = blockIdx.y; pair < n_pairs; pair += gridDim.y)
    match_decide_row(pairs, sides, info, ratio_sqr, first_round, out, total, list_rows, list_unknown, side_cnt, n_sides,
                     pair, row);
}

// Plans the gathered second tensor pass: every side with requested rows gets
// ceil(cnt/128) gather blocks = filter tasks.  A side that does not fit in the
// block budget sends its rows to the full re-scan list instead.
__global__ void k_gather_plan(const TcGatherSide* __restrict__ gsides, int n_sides, const int* __restrict__ side_cnt,
                              const int* __restrict__ list_rows, int block_cap, TcTask* __restrict__ tasks,
                              int* __restrict__ n_blocks, int2* __restrict__ fb_list, int* __restrict__ fb_cnt) {
  const int side = blockIdx.x * blockDim.x + threadIdx.x;
  if (side >= n_sides) return;
  const int cnt = side_cnt[side];
  if (cnt == 0) return;
  const TcGatherSide gs = gsides[side];
  const int nb = (cnt + 127) / 128;
  const int b0 = atomicAdd(n_blocks, nb);
  if (b0 + nb > block_cap) {
    atomicSub(n_blocks, nb);
    const int f0 = atomicAdd(fb_cnt, cnt);
    for (int i = 0; i < cnt; ++i) fb_list[f0 + i] = make_int2(side, list_rows[gs.list_off + i]);
    return;
  }
  for (int i = 0; i < nb; ++i) {
    TcTask t;
    t.q_blk = b0 + i; t.q_row0 = (b0 + i) * 128; t.q_n = min(128, cnt - i * 128);
    t.t_blk0 = gs.t_blk0; t.t_blocks = gs.t_blocks; t.t_n = gs.t_n; t.t_pad = i * 128;
    t.res_off = side;
    tasks[b0 + i] = t;
  }
}

// Exact decision among the candidate columns the filter pass listed for a row: one
// warp per gathered row, one lane per candidate.  The candidate set provably holds
// the true best and second best (every column scoring within 2*eps of the
// approximate second best is in it); rows that overflowed their slots go to the
// full re-scan list.
__global__ void __launch_bounds__(256)
k_exact_cands(const float* __restrict__ desc, const SideMeta* __restrict__ sides, const int* __restrict__ n_blocks,
              const int2* __restrict__ g_meta, const int* __restrict__ cand_cnt, const int* __restrict__ cand,
              RowInfo* __restrict__ info, int2* __restrict__ fb_list, int* __restrict__ fb_cnt) {
  const int lane = threadIdx.x & 31;
  const int nrow = *n_blocks * 128;
  for (int g = blockIdx.x * 8 + (threadIdx.x >> 5); g < nrow; g += gridDim.x * 8) {
    const int2 me = g_meta[g];
    if (me.x < 0) continue;
    const SideMeta sm = sides[me.x];
    const int cnt = cand_cnt[g];
    if (cnt > TC_CAND_CAP || cnt < 1 || (cnt < 2 && sm.t_n >= 2)) {
      if (lane == 0) fb_list[atomicAdd(fb_cnt, 1)] = me;
      continue;
    }
    float mn = FLT_MAX, sec = FLT_MAX;
    int idx = 0x7fffffff;
    if (lane < cnt) {
      idx = cand[(size_t)g * TC_CAND_CAP + lane];
      mn = exact_dist(desc + (size_t)(sm.q_base + me.y) * 128, desc + (size_t)(sm.t_base + idx) * 128);
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
      float m2 = __shfl_xor_sync(0xffffffffu, mn, off);
      float s2 = __shfl_xor_sync(0xffffffffu, sec, off);
      int i2 = __shfl_xor_sync(0xffffffffu, idx, off);
      top2_merge(mn, idx, sec, m2, i2, s2);
    }
    if (lane == 0) {
      RowInfo o; o.mn = mn; o.mn_hi = mn; o.idx = idx; o.sec_lo = sec; o.sec_hi = sec; o.state = 3; o.requested = 1; o.pad = 0;
      info[sm.res_off + me.y] = o;
    }
  }
}

// ------------------------------------------------------------------ result lists on the device
// The decisions are one int per row of the smaller set; what the caller wants is MatchData
// (matcher.hh:14-25): per pair the (i-index, j-index) list in ascending row order.  Counting,
// the prefix over pairs and the ordered compaction run here, so that only the matches themselves
// (8 bytes each) cross PCIe and the host never walks the rows.
// hdr layout (ints): [0] total, [1] undecided rows, [2 .. 2+n) count, [2+n .. 3+2n) offset
__global__ void __launch_bounds__(256)
k_match_count(const PairMeta* __restrict__ pairs, const int* __restrict__ out, int n_pairs, int* __restrict__ hdr) {
  __shared__ int s_c[8], s_p[8];
  const PairMeta pm = pairs[blockIdx.x];
  int c = 0, pend = 0;
  for (int r = pm.k0 + threadIdx.x; r < pm.k1; r += 256) {
    const int v = out[pm.out_off + r];
    c += v >= 0; pend += v == OUT_PENDING;
  }
  for (int off = 16; off; off >>= 1) { c += __shfl_xor_sync(0xffffffffu, c, off); pend += __shfl_xor_sync(0xffffffffu, pend, off); }
  if ((threadIdx.x & 31) == 0) { s_c[threadIdx.x >> 5] = c; s_p[threadIdx.x >> 5] = pend; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int q = 1; q < 8; ++q) { c += s_c[q]; pend += s_p[q]; }
    hdr[2 + blockIdx.x] = c;
    if (pend) atomicAdd(&hdr[1], pend);
  }
}

__global__ void __launch_bounds__(1024)
k_match_offsets(int n_pairs, int* __restrict__ hdr) {
  __shared__ int s_w[32];
  __shared__ int s_carry;
  const int* cnt = hdr + 2;
  int* off = hdr + 2 + n_pairs;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < n_pairs; base += 1024) {
    const int k = base + tid;
    const int v = k < n_pairs ? cnt[k] : 0;
    int incl = v;
    for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
    if (lane == 31) s_w[wid] = incl;
    __syncthreads();
    if (wid == 0) {
      int w = s_w[lane], a = w;
      for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(0xffffffffu, a, d); if (lane >= d) a += t; }
      s_w[lane] = a - w;
    }
    __syncthreads();
    const int carry = s_carry;
    if (k < n_pairs) off[k] = carry + s_w[wid] + incl - v;
    __syncthreads();
    if (tid == 1023) s_carry = carry + s_w[31] + incl;
    __syncthreads();
  }
  if (tid == 0) { off[n_pairs] = s_carry; hdr[0] = s_carry; }
}

__global__ void __launch_bounds__(256)
k_match_write(const PairMeta* __restrict__ pairs, const int* __restrict__ out, int n_pairs, const int* __restrict__ hdr,
              int* __restrict__ dense) {
  __shared__ int s_w[8];
  __shared__ int s_base;
  const PairMeta pm = pairs[blockIdx.x];
  int* dst = dense + 2 * (size_t)hdr[2 + n_pairs + blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) s_base = 0;
  __syncthreads();
  for (int r0 = pm.k0; r0 < pm.k1; r0 += 256) {
    const int r = r0 + tid;
    const int j = r < pm.k1 ? out[pm.out_off + r] : -1;
    const unsigned bal = __ballot_sync(0xffffffffu, j >= 0);
    if (lane == 0) s_w[wid] = __popc(bal);
    __syncthreads();
    int before = s_base;
    for (int q = 0; q < wid; ++q) before += s_w[q];
    if (j >= 0) {
      int* d = dst + 2 * (before + __popc(bal & ((1u << lane) - 1)));
      if (pm.rev) { d[0] = j; d[1] = r; } else { d[0] = r; d[1] = j; }        // MatchData::reverse (matcher.cc:127-128)
    }
    __syncthreads();
    if (tid == 0) { int t = 0; for (int q = 0; q < 8; ++q) t += s_w[q]; s_base += t; }
    __syncthreads();
  }
}

// copies hdr[0] * 2 ints of the dense list (the count lives on the device) into pinned host memory
__global__ void k_match_download(int* __restrict__ h_dst, const int* __restrict__ dense, const int* __restrict__ hdr) {
  const size_t n = (size_t)hdr[0] * 2;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) h_dst[i] = dense[i];
}

// ------------------------------------------------------------------ host driver

struct MatchPlan {
  std::vector<SideMeta> sides;
  std::vector<PairMeta> pairs;
  std::vector<MatchTask> exact_tasks;   // exact path
  std::vector<TcTask> tc_tasks;         // tensor path
  std::vector<int> task_part;           // tensor path: column-range index of each task
  std::vector<TcGatherSide> gsides;     // tensor path: per side, for the gathered second pass
  std::vector<char> rev;                // pair was swapped (first image is the larger set)
  long long res_total = 0, out_total = 0;
  int max_side_n = 0, max_small = 0;
  int parts = 1;                        // first-pass tasks are split into up to this many column ranges
  int shard = 0, n_shards = 1;          // row-sharded call: this call decides share `shard` of every pair's smaller set
  bool lazy = false;                    // columns on demand: no first-pass tasks for the larger sets
  long long large_blocks = 0;           // 128-row blocks of all larger sets
  long long block_pairs = 0;            // sum over pairs of (blocks of the larger set) x (blocks of the smaller set)
};

// counters (ints): [0] matches, then per gather round r < 4: fallback rows, filter blocks, nomination
// blocks; from MC_HEAD on, per decide round and list: requests per side ([round][list][side]).
#define MC_FB(r) (1 + (r))
#define MC_BLK_FILTER(r) (5 + (r))
#define MC_BLK_NOMINATE(r) (9 + (r))
#define MC_HEAD 16
#define MC_ROUNDS 4

static bool use_exact_path() {
  const char* e = getenv("PANO_MATCH_PATH");
  return e && strcmp(e, "exact") == 0;
}

static int build_plan(pano_ctx* ctx, pano_featureset* fs, int n_pairs, const int* ij, MatchPlan& pl,
                      const std::vector<TcImage>* tcimgs) {
  for (int k = 0; k < n_pairs; ++k) {
    int i = ij[2 * k], j = ij[2 * k + 1];
    if (i < 0 || j < 0 || i >= fs->n_images || j >= fs->n_images)
      return ctx_fail(ctx, PANO_ERR_INVALID, "pair %d: image index out of range", k);
    if (fs->h_count[i] > 0 && fs->h_count[j] > 0) {
      const long long bl = (std::max(fs->h_count[i], fs->h_count[j]) + 127) / 128, bs = (std::min(fs->h_count[i], fs->h_count[j]) + 127) / 128;
      pl.large_blocks += bl;
      pl.block_pairs += bl * bs;
    }
  }
  if (tcimgs) {
    // Columns on demand halve the first pass but pay a nomination launch chain in each of three
    // rounds (even when empty): they pay off on large pairs (50 k x 50 k rows = 153 k block pairs)
    // and not on many small ones (13 pairs of ~2.9 k rows = 6.9 k block pairs).
    pl.lazy = pl.block_pairs >= 32768;
    if (const char* e = getenv("PANO_MATCH_LAZY")) pl.lazy = atoi(e) != 0;
    // a shard nominates its own rows of the smaller sets only; whatever it needs of the larger sets
    // (against ALL rows of the smaller set, matcher.cc:57-61) comes on request
    if (pl.n_shards > 1) pl.lazy = true;
    // Tail balance.  The persistent CTAs walk equal tasks round-robin, so n tasks take
    // ceil(n / SMs) task times: a task count just above a multiple of the SM count wastes most of
    // the last wave.
    // Splitting every task into P column ranges (merged in k_refine) makes the waves P times finer.
    long long n1 = 0, tile_sum = 0;       // first-pass tasks, and their target tiles
    for (int k = 0; k < n_pairs; ++k) {
      const int ci = fs->h_count[ij[2 * k]], cj = fs->h_count[ij[2 * k + 1]];
      if (ci <= 0 || cj <= 0) continue;
      const long long bs = (std::min(ci, cj) + 127) / 128, bl = (std::max(ci, cj) + 127) / 128;
      const long long ts = (std::min(ci, cj) + 255) / 256, tl = (std::max(ci, cj) + 255) / 256;
      const long long mine = pl.lazy ? (bs + pl.n_shards - 1) / pl.n_shards : bs;
      n1 += mine; tile_sum += mine * tl;
      if (!pl.lazy) { n1 += bl; tile_sum += bl * ts; }
    }
    const long long W = std::max(1, ctx->num_sms);
    if (n1 > 0 && n1 < 12 * W) {
      // waves x (tiles per part + ~0.7 tile of per-task prologue / merge); split only for a real gain
      const double T = (double)tile_sum / (double)n1;
      auto cost = [&](int P) { return (double)((n1 * P + W - 1) / W) * (T / P + 0.7); };
      double best = cost(1) * 0.96;
      for (int P = 2; P <= 8; ++P)
        if (T / P >= 4.0 && cost(P) < best * 0.99) { best = cost(P); pl.parts = P; }
    }
    if (const char* e = getenv("PANO_MATCH_PARTS")) pl.parts = std::max(1, std::min(8, atoi(e)));
  }
  for (int k = 0; k < n_pairs; ++k) {
    int i = ij[2 * k], j = ij[2 * k + 1];
    // matcher.cc:21-29: loop over the smaller one; rev = l1 > l2
    const bool rev = fs->h_count[i] > fs->h_count[j];
    const int is = rev ? j : i, il = rev ? i : j;
    const int ns = fs->h_count[is], nl = fs->h_count[il];
    // rows [k0, k1) of the smaller set are this call's share (all of them unless row-sharded)
    const int k0 = (int)((long long)ns * pl.shard / pl.n_shards), k1 = (int)((long long)ns * (pl.shard + 1) / pl.n_shards);
    // a part must keep >= 4 target tiles (256 rows each), or its prologue costs more than it balances
    const int tiles_l = tcimgs ? (*tcimgs)[il].n_pad / 256 : 0, tiles_s = tcimgs ? (*tcimgs)[is].n_pad / 256 : 0;
    const int parts_a = std::max(1, std::min(pl.parts, tiles_l / 4)), parts_b = pl.lazy ? 1 : std::max(1, std::min(pl.parts, tiles_s / 4));
    SideMeta a{fs->base[is], fs->base[il], ns, nl, pl.res_total, k0, k1, parts_a, 0}; pl.res_total += ns;
    SideMeta b{fs->base[il], fs->base[is], nl, ns, pl.res_total, 0, nl, parts_b, 0}; pl.res_total += nl;
    PairMeta pm{(int)pl.sides.size(), (int)pl.sides.size() + 1, ns, nl, pl.out_total, rev ? 1 : 0, 0, k0, k1};
    pl.out_total += ns;
    pl.sides.push_back(a); pl.sides.push_back(b);
    pl.pairs.push_back(pm);
    pl.rev.push_back(rev ? 1 : 0);
    pl.max_side_n = std::max(pl.max_side_n, std::max(ns, nl));
    pl.max_small = std::max(pl.max_small, k1 - k0);
    if (tcimgs) {
      const TcImage &ts = (*tcimgs)[is], &tl = (*tcimgs)[il];
      // part p covers target tiles [tiles * p / parts, tiles * (p + 1) / parts); its first column rides
      // in t_pad and its part index is folded into res_off once res_total is known (below)
      auto add_tasks = [&](const TcImage& tq, const TcImage& tt, int row_lo, int row_hi, int q_n, int t_n, long long res_off, int parts) {
        const int tiles = tt.n_pad / 256;
        for (int r0 = row_lo / 128 * 128; r0 < row_hi; r0 += 128)
          for (int pp = 0; pp < parts; ++pp) {
            const int t0 = (int)((long long)tiles * pp / parts), t1 = (int)((long long)tiles * (pp + 1) / parts);
            pl.tc_tasks.push_back(TcTask{tq.blk0 + r0 / 128, r0, q_n, tt.blk0 + 2 * t0, 2 * (t1 - t0), t_n, t0 * 256, res_off});
            pl.task_part.push_back(pp);
          }
      };
      if (nl > 0) add_tasks(ts, tl, k0, k1, ns, nl, a.res_off, parts_a);
      if (ns > 0 && !pl.lazy) add_tasks(tl, ts, 0, nl, nl, ns, b.res_off, parts_b);
      pl.gsides.push_back(TcGatherSide{a.q_base, a.res_off, a.res_off, ts.blk0, tl.blk0, tl.n_pad / 128, nl});
      pl.gsides.push_back(TcGatherSide{b.q_base, b.res_off, b.res_off, tl.blk0, ts.blk0, ts.n_pad / 128, ns});
    } else {
      for (int r0 = k0 / MT * MT; r0 < k1; r0 += MT) pl.exact_tasks.push_back(MatchTask{a.q_base, a.t_base, ns, nl, r0, a.res_off});
      for (int r0 = 0; r0 < nl; r0 += MT) pl.exact_tasks.push_back(MatchTask{b.q_base, b.t_base, nl, ns, r0, b.res_off});
    }
  }
  for (size_t t = 0; t < pl.tc_tasks.size(); ++t) pl.tc_tasks[t].res_off += (long long)pl.task_part[t] * pl.res_total;
  return PANO_OK;
}

struct MatchBuffers {
  DevBuf<unsigned char> tasks; DevBuf<PairMeta> pairs; DevBuf<SideMeta> sides;
  DevBuf<RowInfo> info; DevBuf<TcTop2> approx;
  DevBuf<int2> list;           // full re-scan (fallback) list
  DevBuf<int> counters;        // [0] matches, [1..3] fallback rows per round, [4..6] gather blocks per round,
                               // then side_cnt[round][side]
  int n_counters = 0;
  DevBuf<int> out;
  // gathered second tensor pass
  DevBuf<TcGatherSide> gsides; DevBuf<int> list_rows; DevBuf<TcTask> gtasks; DevBuf<unsigned char> gq;
  DevBuf<int2> g_meta; DevBuf<int> g_thr; DevBuf<int> cand_cnt; DevBuf<int> cand;
  // columns on demand: gathered nomination pass over requested rows that are still unknown
  DevBuf<int> list_unknown; DevBuf<TcTask> ntasks; DevBuf<unsigned char> nq; DevBuf<int2> n_meta;
  DevBuf<TcTop2> n_approx;
  int rounds = 2;              // gather rounds run (the decide after the last one must leave nothing pending)
};

// Runs the plan; leaves per-row decisions in b.out and counters in b.counters.
static int run_plan(pano_ctx* ctx, pano_featureset* fs, const MatchPlan& pl, float ratio, bool tensor,
                    const TcOperands* ops, MatchBuffers& b) {
  int rc = 0;
  const size_t bt = tensor ? pl.tc_tasks.size() * sizeof(TcTask) : pl.exact_tasks.size() * sizeof(MatchTask);
  const size_t bp = pl.pairs.size() * sizeof(PairMeta), bs = pl.sides.size() * sizeof(SideMeta);
  const long long nres = std::max<long long>(pl.res_total, 1);
  if ((rc = b.tasks.alloc(ctx, bt)) || (rc = b.pairs.alloc(ctx, pl.pairs.size())) ||
      (rc = b.sides.alloc(ctx, pl.sides.size())) || (rc = b.info.alloc(ctx, nres)) ||
      (rc = b.approx.alloc(ctx, nres * std::max(pl.parts, 1))) || (rc = b.list.alloc(ctx, nres)) ||
      (rc = b.out.alloc(ctx, std::max<long long>(pl.out_total, 1))))
    return rc;
  const int n_sides = (int)pl.sides.size();
  b.n_counters = MC_HEAD + MC_ROUNDS * 2 * n_sides;
  if ((rc = b.counters.alloc(ctx, b.n_counters))) return rc;
  const void* tsrc = tensor ? (const void*)pl.tc_tasks.data() : (const void*)pl.exact_tasks.data();
  const size_t bg = tensor ? pl.gsides.size() * sizeof(TcGatherSide) : 0;
  if (bg && (rc = b.gsides.alloc(ctx, pl.gsides.size()))) return rc;
  {
    // plan tables + counter reset in one launch
    void* dsts[5] = {b.tasks, b.pairs, b.sides, b.counters, b.gsides};
    const void* srcs[5] = {tsrc, pl.pairs.data(), pl.sides.data(), nullptr, pl.gsides.data()};
    size_t sizes[5] = {bt, bp, bs, b.n_counters * sizeof(int), bg};
    if ((rc = ctx_put_many(ctx, 5, dsts, srcs, sizes))) return rc;
  }
  if (pl.pairs.empty()) return PANO_OK;
  const float rs = ratio * ratio;
  const int n_pairs = (int)pl.pairs.size();
  dim3 gd(std::max(1, ceil_div(pl.max_small, 256)), grid_y(n_pairs));
  if (!tensor) {
    const size_t smem = (size_t)2 * MT * MT_STRIDE * sizeof(float);
    if (!ctx->attr_match) {   // per device, hence per context (see match_tc.cu)
      PANO_CUDA(ctx, cudaFuncSetAttribute(k_match_top2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      ctx->attr_match = true;
    }
    if (!pl.exact_tasks.empty())
      PANO_LAUNCH(ctx, "k_match_top2", k_match_top2, (unsigned)pl.exact_tasks.size(), MT_THREADS, smem, fs->d_desc,
                  (const MatchTask*)b.tasks.get(), b.info);
    if (pl.max_small > 0) {
      if ((rc = b.list_rows.alloc(ctx, nres))) return rc;
      PANO_LAUNCH(ctx, "k_match_decide", k_match_decide, gd, 256, 0, b.pairs, n_pairs, b.sides, b.info, rs, 1, b.out,
                  b.counters, b.list_rows, b.list_rows, b.counters + MC_HEAD, n_sides);
    }
    return PANO_OK;
  }
  rc = tc_run_top2(ctx, ops, (const TcTask*)b.tasks.get(), (int)pl.tc_tasks.size(), b.approx);
  if (rc) return rc;
  if (pl.max_side_n > 0) {
    dim3 gr(ceil_div(pl.max_side_n, 128), grid_y(n_sides));
    PANO_LAUNCH(ctx, "k_refine", k_refine, gr, 128, 0, fs->d_desc, ops->d_norms, ops->d_maxnorm, b.sides, n_sides, b.approx,
                (long long)pl.res_total, rs, pl.lazy ? 1 : 0, b.info);
  }
  if (pl.max_small > 0) {
    // Up to three decide rounds.  A round decides every row it can from the current
    // intervals and lists, per side, the rows it needs exactly (round 1 may need row k
    // itself, round 2 then its column).  Listed rows go through a gathered second
    // tensor pass that enumerates the columns inside each row's error band
    // (k_tc_filter), k_exact_cands takes exact fp32 distances to just those columns,
    // and only rows that overflow their candidate slots are re-scanned against every
    // target (k_exact_rows).
    int block_cap = (int)std::min<size_t>(std::max<size_t>(pl.tc_tasks.size(), 1), 4096);
    if (const char* e = getenv("PANO_MATCH_BLOCK_CAP")) block_cap = std::max(1, std::min(block_cap, atoi(e)));   // test hook: force the full re-scan fallback
    const size_t grow = (size_t)block_cap * 128;
    TcFilter f;
    if ((rc = b.list_rows.alloc(ctx, nres)) || (rc = b.gtasks.alloc(ctx, block_cap)) ||
        (rc = b.gq.alloc(ctx, (size_t)block_cap * tc_block_bytes())) || (rc = b.g_meta.alloc(ctx, grow)) ||
        (rc = b.g_thr.alloc(ctx, grow)) || (rc = b.cand_cnt.alloc(ctx, grow)) ||
        (rc = b.cand.alloc(ctx, grow * TC_CAND_CAP)))
      return rc;
    f.gq = b.gq; f.tasks = b.gtasks; f.gsides = b.gsides; f.list_rows = b.list_rows; f.approx = b.approx;
    f.g_meta = b.g_meta; f.g_thr = b.g_thr; f.cand_cnt = b.cand_cnt; f.cand = b.cand;
    // columns on demand: requested rows that are still unknown get their nomination first
    TcFilter nf;
    int nom_cap = 0;
    if (pl.lazy) {
      nom_cap = (int)std::min<long long>(std::max<long long>(pl.large_blocks, 1), 8192);
      const size_t nrow = (size_t)nom_cap * 128;
      if ((rc = b.list_unknown.alloc(ctx, nres)) || (rc = b.ntasks.alloc(ctx, nom_cap)) ||
          (rc = b.nq.alloc(ctx, (size_t)nom_cap * tc_block_bytes())) || (rc = b.n_meta.alloc(ctx, nrow)) ||
          (rc = b.n_approx.alloc(ctx, nrow)))
        return rc;
      nf.gq = b.nq; nf.tasks = b.ntasks; nf.gsides = b.gsides; nf.list_rows = b.list_unknown; nf.approx = nullptr;
      nf.g_meta = b.n_meta; nf.g_thr = nullptr; nf.cand_cnt = nullptr; nf.cand = nullptr;
    }
    int* list_unknown = pl.lazy ? b.list_unknown : b.list_rows;   // never written when nothing is unknown
    const int eg = ctx->num_sms * 4;
    // A row may need: its own exact top-2 (filter), then the nomination of a column it only now
    // knows, then that column's exact top-2 — one more round than when every column starts nominated.
    b.rounds = pl.lazy ? 3 : 2;
    for (int round = 0; round <= b.rounds; ++round) {
      int* side_cnt = b.counters + MC_HEAD + round * 2 * n_sides;
      int* fb_cnt = b.counters + MC_FB(round);
      int* n_blocks = b.counters + MC_BLK_FILTER(round);
      PANO_LAUNCH(ctx, "k_match_decide", k_match_decide, gd, 256, 0, b.pairs, n_pairs, b.sides, b.info, rs, round == 0 ? 1 : 0,
                  b.out, b.counters, b.list_rows, list_unknown, side_cnt, n_sides);
      if (round == b.rounds) break;
      if (pl.lazy) {
        int* nom_blocks = b.counters + MC_BLK_NOMINATE(round);
        PANO_LAUNCH(ctx, "k_gather_plan", k_gather_plan, ceil_div(n_sides, 128), 128, 0, b.gsides, n_sides,
                    side_cnt + n_sides, b.list_unknown, nom_cap, b.ntasks, nom_blocks, b.list, fb_cnt);
        nf.n_tasks = nom_blocks;
        if ((rc = tc_run_nominate(ctx, ops, &nf, nom_cap, b.n_approx))) return rc;
        PANO_LAUNCH(ctx, "k_refine_gathered", k_refine_gathered, nom_cap, 128, 0, fs->d_desc, ops->d_norms, ops->d_maxnorm,
                    b.sides, b.n_meta, b.n_approx, nom_blocks, rs, b.approx, b.info);
      }
      PANO_LAUNCH(ctx, "k_gather_plan", k_gather_plan, ceil_div(n_sides, 128), 128, 0, b.gsides, n_sides, side_cnt,
                  b.list_rows, block_cap, b.gtasks, n_blocks, b.list, fb_cnt);
      f.n_tasks = n_blocks;
      if ((rc = tc_run_filter(ctx, ops, &f, block_cap))) return rc;
      PANO_LAUNCH(ctx, "k_exact_cands", k_exact_cands, eg, 256, 0, fs->d_desc, b.sides, n_blocks, b.g_meta, b.cand_cnt,
                  b.cand, b.info, b.list, fb_cnt);
      PANO_LAUNCH(ctx, "k_exact_rows", k_exact_rows, eg, 256, 0, fs->d_desc, b.sides, b.list, fb_cnt, b.info);
    }
  }
  return PANO_OK;
}

static int ensure_tc_operands(pano_ctx* ctx, pano_featureset* fs, std::vector<TcImage>& imgs) {
  imgs.resize(fs->n_images);
  int blk = 0;
  for (int i = 0; i < fs->n_images; ++i) {
    TcImage& im = imgs[i];
    im.row0 = fs->base[i]; im.n = fs->h_count[i];
    im.n_pad = (im.n + 255) / 256 * 256;
    im.blk0 = blk;
    blk += im.n_pad / 128;
  }
  if (fs->tc_ready) return PANO_OK;
  int rc = tc_prepare(ctx, fs->d_desc, imgs, &fs->tc);
  if (rc) return rc;
  fs->tc_ready = true;
  return PANO_OK;
}

static int match_common(pano_ctx* ctx, pano_featureset* fs, int n_pairs, const int* ij, const pano_params* p,
                        int shard, int n_shards, MatchPlan& pl, MatchBuffers& b) {
  if (n_shards < 1 || shard < 0 || shard >= n_shards) return ctx_fail(ctx, PANO_ERR_INVALID, "shard %d of %d", shard, n_shards);
  pl.shard = shard; pl.n_shards = n_shards;
  int rc = featureset_sync_counts(fs);
  if (rc) return rc;
  const bool tensor = !use_exact_path();
  std::vector<TcImage> tcimgs;
  if (tensor && (rc = ensure_tc_operands(ctx, fs, tcimgs))) return rc;
  rc = build_plan(ctx, fs, n_pairs, ij, pl, tensor ? &tcimgs : nullptr);
  if (rc) return rc;
  return run_plan(ctx, fs, pl, p->match_reject_next_ratio, tensor, &fs->tc, b);
}

extern "C" {

int pano_match_pairs(pano_ctx* ctx, pano_featureset* fs, int n_pairs, const int* ij, const pano_params* p,
                     pano_matches* out) {
  return pano_match_pairs_shard(ctx, fs, n_pairs, ij, p, 0, 1, out);
}

int pano_match_pairs_shard(pano_ctx* ctx, pano_featureset* fs, int n_pairs, const int* ij, const pano_params* p,
                           int shard, int n_shards, pano_matches* out) {
  ctx_enter(ctx);
  if (!ctx || !fs || !out || n_pairs < 0 || (n_pairs && !ij) || !p) return PANO_ERR_INVALID;
  memset(out, 0, sizeof(*out));
  MatchPlan pl;
  MatchBuffers b;
  int rc = match_common(ctx, fs, n_pairs, ij, p, shard, n_shards, pl, b);
  if (rc) return rc;
  // count -> offsets -> ordered compaction on the device; one read-back of header + matches
  const size_t n_hdr = 3 + 2 * (size_t)n_pairs;
  const size_t cap = (size_t)std::max<long long>(pl.out_total, 1) * 2;
  DevBuf<int> d_hdr, d_dense;
  if ((rc = d_hdr.alloc(ctx, n_hdr)) || (rc = d_dense.alloc(ctx, cap))) return rc;
  int* h_stage = (int*)ctx_ring(ctx, (n_hdr + cap) * sizeof(int));
  if (!h_stage) return ctx_fail(ctx, PANO_ERR_CUDA, "pinned ring allocation failed");
  if ((rc = ctx_zero(ctx, d_hdr, 2 * sizeof(int)))) return rc;
  if (n_pairs > 0) {
    PANO_LAUNCH(ctx, "k_match_count", k_match_count, n_pairs, 256, 0, b.pairs, b.out, n_pairs, d_hdr);
    PANO_LAUNCH(ctx, "k_match_offsets", k_match_offsets, 1, 1024, 0, n_pairs, d_hdr);
    PANO_LAUNCH(ctx, "k_match_write", k_match_write, n_pairs, 256, 0, b.pairs, b.out, n_pairs, d_hdr, d_dense);
    PANO_LAUNCH(ctx, "k_match_download", k_match_download, std::max(1, std::min(ctx->num_sms, (int)(cap / 4096) + 1)), 256, 0,
                h_stage + n_hdr, d_dense, d_hdr);
  }
  rc = ctx_store(ctx, h_stage, d_hdr, n_hdr * sizeof(int));
  cudaError_t e = ctx_spin_stream(ctx);
  if (rc) return rc;
  if (e != cudaSuccess) return ctx_cuda(ctx, e, "match download");
  if (n_pairs > 0 && h_stage[1] != 0) return ctx_fail(ctx, PANO_ERR_CUDA, "match: %d undecided rows (internal error)", h_stage[1]);
  const int total = n_pairs > 0 ? h_stage[0] : 0;
  out->n_pairs = n_pairs;
  out->count = (int*)calloc(std::max(n_pairs, 1), sizeof(int));
  out->offset = (int*)calloc(n_pairs + 1, sizeof(int));
  out->idx = (int*)calloc((size_t)std::max(total, 1) * 2, sizeof(int));
  if (n_pairs > 0) {
    memcpy(out->count, h_stage + 2, (size_t)n_pairs * sizeof(int));
    memcpy(out->offset, h_stage + 2 + n_pairs, (size_t)(n_pairs + 1) * sizeof(int));
    memcpy(out->idx, h_stage + n_hdr, (size_t)total * 2 * sizeof(int));
  }
  return PANO_OK;
}

void pano_matches_free(pano_matches* m) {
  if (!m) return;
  free(m->count); free(m->offset); free(m->idx);
  memset(m, 0, sizeof(*m));
}

int pano_match_pairs_dev(pano_ctx* ctx, pano_featureset* fs, int n_pairs, const int* ij, const pano_params* p,
                         int* total_matches) {
  return pano_match_pairs_dev_shard(ctx, fs, n_pairs, ij, p, 0, 1, total_matches);
}

int pano_match_pairs_dev_shard(pano_ctx* ctx, pano_featureset* fs, int n_pairs, const int* ij, const pano_params* p,
                               int shard, int n_shards, int* total_matches) {
  ctx_enter(ctx);
  if (!ctx || !fs || n_pairs < 0 || (n_pairs && !ij) || !p || !total_matches) return PANO_ERR_INVALID;
  MatchPlan pl;
  MatchBuffers b;
  int rc = match_common(ctx, fs, n_pairs, ij, p, shard, n_shards, pl, b);
  if (rc) return rc;
  int* h = (int*)ctx_ring(ctx, (size_t)std::max(b.n_counters, MC_HEAD) * sizeof(int));
  if (!h) return ctx_fail(ctx, PANO_ERR_CUDA, "pinned ring allocation failed");
  const int n_counters = b.n_counters, n_sides = (int)pl.sides.size(), rounds = b.rounds;
  rc = b.counters ? ctx_store(ctx, h, b.counters, (size_t)n_counters * sizeof(int)) : 0;
  cudaError_t e = ctx_spin_stream(ctx);
  if (rc) return rc;
  if (e != cudaSuccess) return ctx_cuda(ctx, e, "match total download");
  if (n_counters < MC_HEAD) { *total_matches = 0; return PANO_OK; }
  long long requested = 0, nominated = 0, undecided = 0, rescans = 0;
  for (int round = 0; round <= rounds; ++round)
    for (int q = 0; q < 2 * n_sides; ++q) {
      const int v = h[MC_HEAD + round * 2 * n_sides + q];
      if (round == rounds) undecided += v;
      else if (q < n_sides) requested += v;      // rows that went through the exact (filter) pass
      else nominated += v;                       // columns on demand: rows nominated on request
    }
  for (int round = 0; round < rounds; ++round) rescans += h[MC_FB(round)];
  ctx->last_match_nominated_rows = (int)nominated;
  ctx->last_match_exact_rows = (int)requested;
  ctx->last_match_full_rescans = (int)rescans;
  if (undecided != 0) return ctx_fail(ctx, PANO_ERR_CUDA, "match: %lld rows undecided after the exact passes", undecided);
  *total_matches = h[0];
  return PANO_OK;
}

int pano_match_bruteforce(pano_ctx* ctx, const float* a, int n, const float* b, int m, const pano_params* p,
                          int* pairs_out, int* n_pairs_out) {
  ctx_enter(ctx);
  if (!ctx || n < 0 || m < 0 || !p || !pairs_out || !n_pairs_out) return PANO_ERR_INVALID;
  *n_pairs_out = 0;
  if (n == 0 || m == 0) return PANO_OK;
  int cnt[2] = {n, m};
  const float* ds[2] = {a, b};
  pano_featureset* fs = nullptr;
  int rc = pano_featureset_upload(ctx, 2, cnt, ds, nullptr, &fs);
  if (rc) return rc;
  int ij[2] = {0, 1};
  pano_matches mt;
  rc = pano_match_pairs(ctx, fs, 1, ij, p, &mt);
  pano_featureset_free(fs);
  if (rc) return rc;
  *n_pairs_out = mt.count[0];
  memcpy(pairs_out, mt.idx, sizeof(int) * 2 * mt.count[0]);
  pano_matches_free(&mt);
  return PANO_OK;
}

}  // extern "C"
