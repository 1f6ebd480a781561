// ba.cu — bundle-adjustment Jacobian assembly on the device (SURVEY.md §8f.4), and the session
// that keeps one LM iteration's per-point work on the device (residuals, avg / max, J, J^T J, b;
// see the second half of the file).
//
// Replaces the per-point part of IncrementalBundleAdjuster::calcJacobianSymbolic
// (stitch/incremental_bundle_adjuster.cc:306-383): for every point match of every image pair
// the 2 x 12 block of d(residual)/d(camera parameters) (two rows of J, :355-361) and the
// running sums of J^T J (:363-382).  "J.rows() could reach 700000" (:280): the rows are
// independent, the J^T J entries are independent chains.  What stays on the host is the
// per-PAIR algebra in front of the loop (:288-304 and the loop-invariant 3x3 products inside
// it): those go through Homography::operator* / inverse and Camera::rotation_to_angle, which
// are Eigen calls in the reference — the caller evaluates them with its own Eigen and hands
// the 13 matrices per pair in (pano_ba_pair, include/pano_b200.h).
//
// Arithmetic is the reference's, operation for operation, in f64 without contraction:
// Homography::trans (homography.hh:52-57) sums its three products left to right;
// `sqr(homo.z)` is lib/utils.hh:25's FLOAT sqr (the double is narrowed first); drdv is the
// macro at :316-319.  Every J^T J entry is one sequential sum over pairs in list order and
// points in match order — exactly the order `JtJ(i1, i2) += val` runs in — so the result is
// bit-identical, not merely close.
#include "common.cuh"
#include <string.h>
#include <vector>

struct BaPairDev {
  int from, to, match_begin, n_match;
  double m[13][9];
};

struct BaVec { double x, y, z; };

__device__ __forceinline__ BaVec ba_trans(const double* __restrict__ d, BaVec v) {   // Homography::trans(const Vec&)
  BaVec r;
  r.x = d[0] * v.x + d[1] * v.y + d[2] * v.z;
  r.y = d[3] * v.x + d[4] * v.y + d[5] * v.z;
  r.z = d[6] * v.x + d[7] * v.y + d[8] * v.z;
  return r;
}

// the three constant matrices dK/dfocal, dK/dppx, dK/dppy (:84-95), applied with the same full products
__constant__ double c_dKd[3][9] = {{1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0},
                                   {0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0},
                                   {0.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0}};

// pair matrices (order fixed by the header): 0 Hto_to_from; 1 R_from*toRinv*toKinv; 2 toRinv*toKinv;
// 3..5 fromK*dRfromdvi[k]; 6 toKinv; 7..9 m*dKd{focal,ppx,ppy}, m = fromK*R_from*toRinv*toKinv;
// 10..12 (fromK*R_from)*dRtodviT[k]
__global__ void __launch_bounds__(128)
k_ba_rows(const BaPairDev* __restrict__ pairs, int n_pair, const double2* __restrict__ pts_to, double* __restrict__ rows) {
  __shared__ double s_m[13][9];
  // pairs on gridDim.y (at most 65,535): the blocks of a y index take every gridDim.y-th pair
  for (int p = blockIdx.y; p < n_pair; p += gridDim.y) {
    const BaPairDev& pr = pairs[p];
    __syncthreads();                                     // the previous pair's matrices are no longer read
    for (int q = threadIdx.x; q < 13 * 9; q += blockDim.x) s_m[q / 9][q % 9] = pr.m[q / 9][q % 9];
    __syncthreads();
    const int n = pr.n_match, begin = pr.match_begin;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
      const double2 to = pts_to[begin + i];
      const BaVec tov{to.x, to.y, 1.0};                    // trans(Vec2D) = trans(Vec(x, y, 1))
      const BaVec homo = ba_trans(s_m[0], tov);
      const float hzf = (float)homo.z;                     // sqr(float), lib/utils.hh:25
      const double hz_sqr_inv = 1.0 / (double)(hzf * hzf);
      const double hz_inv = 1.0 / homo.z;
      double* out = rows + (size_t)(begin + i) * 24;       // row idx: dfrom.x[6], dto.x[6]; row idx+1: dfrom.y[6], dto.y[6]
      auto drdv = [&](BaVec dhdv, int col) {
        out[col] = -dhdv.x * hz_inv + dhdv.z * homo.x * hz_sqr_inv;
        out[12 + col] = -dhdv.y * hz_inv + dhdv.z * homo.y * hz_sqr_inv;
      };
      BaVec dot_u2 = ba_trans(s_m[1], tov);
#pragma unroll
      for (int k = 0; k < 3; ++k) drdv(ba_trans(c_dKd[k], dot_u2), k);            // dfrom: focal, ppx, ppy
      dot_u2 = ba_trans(s_m[2], tov);
#pragma unroll
      for (int k = 0; k < 3; ++k) drdv(ba_trans(s_m[3 + k], dot_u2), 3 + k);       // dfrom: rotation
      const BaVec ku = ba_trans(s_m[6], tov);
      dot_u2 = BaVec{ku.x * -1.0, ku.y * -1.0, ku.z * -1.0};                       // Vec::operator*(-1)
#pragma unroll
      for (int k = 0; k < 3; ++k) drdv(ba_trans(s_m[7 + k], dot_u2), 6 + k);       // dto: focal, ppx, ppy
#pragma unroll
      for (int k = 0; k < 3; ++k) drdv(ba_trans(s_m[10 + k], ku), 9 + k);          // dto: rotation
    }
  }
}

// One CTA per 6x6 block (a, b) of J^T J, one thread per entry (i, j).  The pair list is walked in
// order; a pair contributes to this block as the cross term (from=a, to=b: dfrom[i].dto[j]), its
// mirror (from=b, to=a: JtJ(i2, i1) += dfrom[i'].dto[j'] with i'=j, j'=i), or a diagonal term
// (a == b == from: dfrom[i].dfrom[j]; a == b == to: dto[i].dto[j]).  Vec2D::dot = x*v.x + y*v.y.
__global__ void __launch_bounds__(64)
k_ba_jtj(const BaPairDev* __restrict__ pairs, int n_pair, int n_cam, const double* __restrict__ rows,
         double* __restrict__ jtj) {
  const int a = blockIdx.y, b = blockIdx.x, t = threadIdx.x;
  if (t >= 36) return;
  const int i = t / 6, j = t % 6;
  double acc = 0.0;                                       // JtJ.setZero()
  for (int p = 0; p < n_pair; ++p) {
    const int from = pairs[p].from, to = pairs[p].to;
    int c0, c1;                                           // columns of the compact row whose 2-vectors are multiplied
    if (a == from && b == to) { c0 = i; c1 = 6 + j; }
    else if (a == to && b == from) { c0 = j; c1 = 6 + i; }
    else if (a == b && a == from) { c0 = i; c1 = j; }
    else if (a == b && a == to) { c0 = 6 + i; c1 = 6 + j; }
    else continue;
    const double* r = rows + (size_t)pairs[p].match_begin * 24;
    const int n = pairs[p].n_match;
    for (int k = 0; k < n; ++k, r += 24) {
      const double val = r[c0] * r[c1] + r[12 + c0] * r[12 + c1];
      acc += val;
    }
  }
  const size_t N = (size_t)n_cam * 6;
  jtj[(size_t)(a * 6 + i) * N + (size_t)b * 6 + j] = acc;
}

extern "C" int pano_ba_jacobian(pano_ctx* ctx, int n_cam, int n_pair, const pano_ba_pair* pairs, const double* pts_to,
                                double* j_rows, double* jtj) {
  ctx_enter(ctx);
  if (!ctx || n_cam <= 0 || n_pair < 0 || (n_pair && (!pairs || !pts_to)) || !jtj) return PANO_ERR_INVALID;
  if (n_cam > PANO_MAX_IMAGES)   // J^T J blocks on (gridDim.x, gridDim.y)
    return ctx_fail(ctx, PANO_ERR_INVALID, "ba: %d cameras (limit %d)", n_cam, PANO_MAX_IMAGES);
  static_assert(sizeof(BaPairDev) == sizeof(pano_ba_pair), "pano_ba_pair layout");
  long long nm = 0;
  int max_match = 0;
  for (int k = 0; k < n_pair; ++k) {
    const pano_ba_pair& p = pairs[k];
    if (p.from < 0 || p.from >= n_cam || p.to < 0 || p.to >= n_cam || p.from == p.to || p.n_match < 0 || p.match_begin != nm)
      return ctx_fail(ctx, PANO_ERR_INVALID, "ba: pair %d has a camera slot out of range or a match range that does not follow the previous pair's", k);
    nm += p.n_match;
    max_match = std::max(max_match, p.n_match);
  }
  const size_t N = (size_t)n_cam * 6;
  const size_t b_pairs = align_up((size_t)n_pair * sizeof(BaPairDev), 16), b_pts = (size_t)nm * 16;   // double2 loads behind the pair table
  const size_t b_rows = (size_t)nm * 24 * sizeof(double), b_jtj = N * N * sizeof(double);
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));            // the staging buffers may still feed earlier copies
  char* st = (char*)ctx_pinned(ctx, b_pairs + b_pts + 64);
  char* so = (char*)ctx_pinned2(ctx, (j_rows ? b_rows : 0) + b_jtj + 64);
  if (!st || !so) return ctx_fail(ctx, PANO_ERR_CUDA, "ba: pinned staging allocation failed");
  if (n_pair) memcpy(st, pairs, (size_t)n_pair * sizeof(BaPairDev));
  if (b_pts) memcpy(st + b_pairs, pts_to, b_pts);
  DevBuf<char> d_in, d_out;
  int rc = d_in.alloc(ctx, b_pairs + b_pts + 64);
  if (!rc) rc = d_out.alloc(ctx, b_rows + b_jtj + 64);
  if (rc) return rc;
  PANO_CUDA(ctx, cudaMemcpyAsync(d_in, st, b_pairs + b_pts, cudaMemcpyHostToDevice, ctx->stream));
  const BaPairDev* d_pairs = (const BaPairDev*)d_in.get();
  const double2* d_pts = (const double2*)(d_in + b_pairs);
  double* d_rows = (double*)d_out.get();
  double* d_jtj = (double*)(d_out + b_rows);
  if (n_pair && max_match) {
    dim3 grid((unsigned)std::max(1, std::min((max_match + 127) / 128, 1024)), grid_y(n_pair));
    PANO_LAUNCH(ctx, "k_ba_rows", k_ba_rows, grid, 128, 0, d_pairs, n_pair, d_pts, d_rows);
  }
  dim3 gj((unsigned)n_cam, (unsigned)n_cam);
  PANO_LAUNCH(ctx, "k_ba_jtj", k_ba_jtj, gj, 64, 0, d_pairs, n_pair, n_cam, d_rows, d_jtj);
  if (j_rows && b_rows) PANO_CUDA(ctx, cudaMemcpyAsync(so, d_rows, b_rows, cudaMemcpyDeviceToHost, ctx->stream));
  PANO_CUDA(ctx, cudaMemcpyAsync(so + (j_rows ? b_rows : 0), d_jtj, b_jtj, cudaMemcpyDeviceToHost, ctx->stream));
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (j_rows && b_rows) memcpy(j_rows, so, b_rows);
  memcpy(jtj, so + (j_rows ? b_rows : 0), b_jtj);
  return PANO_OK;
}

// ------------------------------------------------------------------ LM-iteration session
// The rest of one LM iteration's per-point work (IncrementalBundleAdjuster::optimize,
// incremental_bundle_adjuster.cc:117-169): calcError (:171-197) with ErrorStats::update_stats
// (:199-220), and b = J^T * err_vec (:237-238), next to the J / J^T J of k_ba_rows / k_ba_jtj.
// The match coordinates, J and the last residual vector stay on the device between calls, so an
// iteration moves only the per-pair matrices up and J^T J, b, avg and max down.

struct BaErrStats {
  unsigned long long max_bits;   // bit pattern of the largest non-NaN |r| (non-negative doubles order like their bits)
};

// calcError's loop (:180-195): transformed = Hto_to_from.trans2d(to) (homography.hh:53-64), r = from - transformed;
// also the FLOAT squares update_stats sums (error_func = sqr(diff), lib/utils.hh:25's float overload).
__global__ void __launch_bounds__(128)
k_ba_residuals(const BaPairDev* __restrict__ pairs, int n_pair, const double* __restrict__ hto,
               const double2* __restrict__ pts_to, const double2* __restrict__ pts_from, double2* __restrict__ res, float2* __restrict__ sq,
               BaErrStats* __restrict__ st, int* __restrict__ pair_nonfinite) {
  __shared__ double s_h[9];
  // pairs on gridDim.y (at most 65,535): the blocks of a y index take every gridDim.y-th pair
  for (int p = blockIdx.y; p < n_pair; p += gridDim.y) {
    __syncthreads();                                      // the previous pair's matrix is no longer read
    if (threadIdx.x < 9) s_h[threadIdx.x] = hto[(size_t)p * 9 + threadIdx.x];
    __syncthreads();
    const int n = pairs[p].n_match, begin = pairs[p].match_begin;
    unsigned long long mx = 0ull;                           // update_max(max, fabs(e)) from max = 0
    bool bad = false;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
      const double2 to = pts_to[begin + i], fr = pts_from[begin + i];
      const BaVec t = ba_trans(s_h, BaVec{to.x, to.y, 1.0});
      const double denom = 1.0 / t.z;                       // trans_normalize
      const double rx = fr.x - t.x * denom, ry = fr.y - t.y * denom;
      res[begin + i] = make_double2(rx, ry);
      const float fx = (float)rx, fy = (float)ry;
      sq[begin + i] = make_float2(fx * fx, fy * fy);
      bad |= !isfinite(rx) || !isfinite(ry);
      const double ax = fabs(rx), ay = fabs(ry);            // dest < NaN is false: NaN never becomes the max
      if (!isnan(ax)) mx = max(mx, (unsigned long long)__double_as_longlong(ax));
      if (!isnan(ay)) mx = max(mx, (unsigned long long)__double_as_longlong(ay));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    bad = __any_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0) {
      if (mx) atomicMax(&st->max_bits, mx);
      if (bad) atomicOr(&pair_nonfinite[p], 1);
    }
  }
}

// update_stats' avg (:211-218): the squares summed one after the other in residual order into a double,
// divided by residuals.size(), sqrt.  The chain cannot be split without changing bits, so one thread adds;
// the block stages the next chunk into shared memory with coalesced loads while it does.
// Writes {avg, max} to host-mapped memory.
constexpr int kBaSumChunk = 4096;
__global__ void __launch_bounds__(1024)
k_ba_error_sum(const float* __restrict__ sq, long long n_res, const BaErrStats* __restrict__ st, double* out) {
  __shared__ __align__(16) float buf[2][kBaSumChunk];
  const int tid = threadIdx.x;
  const long long n_chunk = (n_res + kBaSumChunk - 1) / kBaSumChunk;
  double acc = 0.0;                                       // avg = 0
  for (int k = tid; k < kBaSumChunk && k < n_res; k += blockDim.x) buf[0][k] = sq[k];
  __syncthreads();
  for (long long c = 0; c < n_chunk; ++c) {
    if (c + 1 < n_chunk) {
      const long long base = (c + 1) * kBaSumChunk;
      float* nb = buf[(c + 1) & 1];
      for (int k = tid; k < kBaSumChunk && base + k < n_res; k += blockDim.x) nb[k] = sq[base + k];
    }
    if (tid == 0) {
      const long long len = min((long long)kBaSumChunk, n_res - c * kBaSumChunk);
      const float4* b4 = reinterpret_cast<const float4*>(buf[c & 1]);
      int k = 0;
#pragma unroll 8
      for (; k + 4 <= len; k += 4) {
        const float4 v = b4[k >> 2];
        acc += (double)v.x; acc += (double)v.y; acc += (double)v.z; acc += (double)v.w;
      }
      for (; k < len; ++k) acc += (double)buf[c & 1][k];
    }
    __syncthreads();
  }
  if (tid == 0) {
    acc /= (double)n_res;                                 // avg /= residuals.size(): 0 / 0 = NaN without matches
    out[0] = sqrt(acc);
    out[1] = __longlong_as_double((long long)st->max_bits);
  }
}

// b = J^T * err_vec (:237-238), one CTA per column of J: one sequential sum over J's rows in row order
// (x row, then y row of every match), each product rounded on its own.  Only the pairs that have the
// column's camera as `from` or `to` hold non-zero entries; skipping the others adds +0 exactly, unless one
// of their residuals is not finite: 0 * inf = NaN, and the entry is NaN.  (The camera's own pairs are in
// the chain, so their inf residuals give what the reference's sum gives: +-inf or NaN.)
// The products are independent: the CTA forms a chunk of them in shared memory while thread 0 adds the
// previous chunk, so the column costs one dependent add per product instead of a global load each.
constexpr int kBaJtrChunk = 1024;                         // matches per chunk (2 products each)
__global__ void __launch_bounds__(128)
k_ba_jtr(const BaPairDev* __restrict__ pairs, int n_pair, const double* __restrict__ rows,
         const double* __restrict__ res, const int* __restrict__ pair_nonfinite, double* __restrict__ b) {
  __shared__ double buf[2][2 * kBaJtrChunk];
  const int col = blockIdx.x, cam = col / 6, j = col % 6, tid = threadIdx.x;
  double acc = 0.0;
  bool zero_times_nonfinite = false;
  int cur = 0, pending = 0;                               // buf[cur ^ 1] holds `pending` products to add
  for (int p = 0; p < n_pair; ++p) {
    int c;
    if (pairs[p].from == cam) c = j;
    else if (pairs[p].to == cam) c = 6 + j;
    else { zero_times_nonfinite |= pair_nonfinite[p] != 0; continue; }
    const int begin = pairs[p].match_begin, n = pairs[p].n_match;
    for (int k0 = 0; k0 < n; k0 += kBaJtrChunk) {
      const int len = min(kBaJtrChunk, n - k0);
      double* out = buf[cur];
      for (int k = tid; k < len; k += blockDim.x) {
        const size_t m = (size_t)begin + k0 + k;
        const double2 e = reinterpret_cast<const double2*>(res)[m];
        out[2 * k] = rows[m * 24 + c] * e.x;
        out[2 * k + 1] = rows[m * 24 + 12 + c] * e.y;
      }
      if (tid == 0) {
        const double* in = buf[cur ^ 1];
#pragma unroll 8
        for (int q = 0; q < pending; ++q) acc += in[q];
      }
      __syncthreads();
      pending = 2 * len;
      cur ^= 1;
    }
  }
  if (tid == 0) {
    const double* in = buf[cur ^ 1];
    for (int q = 0; q < pending; ++q) acc += in[q];
    b[col] = zero_times_nonfinite ? __longlong_as_double(0x7ff8000000000000ll) : acc;
  }
}

struct pano_ba_session {
  ~pano_ba_session() {
    cudaStreamSynchronize(ctx->stream);   // h_out may still be written by a queued kernel
    ctx_small_pinned_put(ctx, std::move(h_out));
  }
  pano_ctx* ctx = nullptr;
  int n_cam = 0, n_pair = 0, max_match = 0;
  long long nm = 0;
  bool have_error = false;                 // residuals of a pano_ba_error call are on the device
  std::vector<BaPairDev> table;            // links + the matrices of the last pano_ba_normal_equations
  DevBuf<char> arena;
  BaPairDev* d_pairs = nullptr;
  double2 *d_to = nullptr, *d_from = nullptr, *d_res = nullptr;
  double *d_rows = nullptr, *d_hto = nullptr, *d_jtj = nullptr, *d_b = nullptr;
  float2* d_sq = nullptr;
  BaErrStats* d_st = nullptr;
  int* d_nonfinite = nullptr;              // per pair: one of its residuals is inf or NaN
  PinnedBuf h_out;                         // host-mapped {avg, max}
};

extern "C" int pano_ba_session_create(pano_ctx* ctx, int n_cam, int n_pair, const pano_ba_link* links, const double* pts,
                                      pano_ba_session** out) {
  if (out) *out = nullptr;
  if (!ctx || !out || n_cam <= 0 || n_pair < 0 || (n_pair && !links)) return PANO_ERR_INVALID;
  ctx_enter(ctx);
  if (n_cam > PANO_MAX_IMAGES)   // J^T J blocks on (gridDim.x, gridDim.y)
    return ctx_fail(ctx, PANO_ERR_INVALID, "ba session: %d cameras (limit %d)", n_cam, PANO_MAX_IMAGES);
  long long nm = 0;
  int max_match = 0;
  for (int k = 0; k < n_pair; ++k) {
    const pano_ba_link& p = links[k];
    if (p.from < 0 || p.from >= n_cam || p.to < 0 || p.to >= n_cam || p.from == p.to || p.n_match < 0 || p.match_begin != nm)
      return ctx_fail(ctx, PANO_ERR_INVALID, "ba session: pair %d has a camera slot out of range or a match range that does not follow the previous pair's", k);
    nm += p.n_match;
    max_match = std::max(max_match, p.n_match);
  }
  if (nm && !pts) return ctx_fail(ctx, PANO_ERR_INVALID, "ba session: %lld matches but no coordinates", nm);
  if (2 * nm > 0x7fffffffll) return ctx_fail(ctx, PANO_ERR_INVALID, "ba session: %lld matches is too many", nm);
  std::unique_ptr<pano_ba_session> s(new pano_ba_session);
  s->ctx = ctx; s->n_cam = n_cam; s->n_pair = n_pair; s->nm = nm; s->max_match = max_match;
  s->table.resize(n_pair);
  for (int k = 0; k < n_pair; ++k) {
    memset(&s->table[k], 0, sizeof(BaPairDev));
    s->table[k].from = links[k].from; s->table[k].to = links[k].to;
    s->table[k].match_begin = links[k].match_begin; s->table[k].n_match = links[k].n_match;
  }
  const size_t N = (size_t)n_cam * 6;
  const size_t b_pairs = align_up((size_t)n_pair * sizeof(BaPairDev) + 16, 256), b_pts = align_up((size_t)nm * 16 + 16, 256);
  const size_t b_rows = align_up((size_t)nm * 24 * 8 + 16, 256), b_sq = align_up((size_t)nm * 8 + 16, 256);
  const size_t b_hto = align_up((size_t)n_pair * 72 + 16, 256), b_jtj = align_up(N * N * 8, 256), b_b = align_up(N * 8, 256);
  const size_t b_st = 256, b_flags = align_up((size_t)n_pair * 4 + 16, 256);
  const size_t total = b_pairs + 3 * b_pts + b_rows + b_sq + b_hto + b_jtj + b_b + b_st + b_flags;
  int rc = s->arena.alloc(ctx, total);
  if (rc) return rc;
  char* q = s->arena;
  s->d_pairs = (BaPairDev*)q; q += b_pairs;
  s->d_to = (double2*)q; q += b_pts;
  s->d_from = (double2*)q; q += b_pts;
  s->d_res = (double2*)q; q += b_pts;
  s->d_rows = (double*)q; q += b_rows;
  s->d_sq = (float2*)q; q += b_sq;
  s->d_hto = (double*)q; q += b_hto;
  s->d_jtj = (double*)q; q += b_jtj;
  s->d_b = (double*)q; q += b_b;
  s->d_st = (BaErrStats*)q; q += b_st;
  s->d_nonfinite = (int*)q;
  s->h_out = ctx_small_pinned_get(ctx, 64);
  if (!s->h_out.get()) return ctx_fail(ctx, PANO_ERR_CUDA, "ba session: pinned allocation failed");
  // one-time upload of the pair table and the coordinates, split into p.first (to) and p.second (from)
  const size_t up = (size_t)n_pair * sizeof(BaPairDev) + (size_t)nm * 32;
  if (up) {
    cudaError_t e = cudaStreamSynchronize(ctx->stream);  // the staging buffer may still feed earlier copies
    char* st = (char*)ctx_pinned(ctx, up + 64);
    if (e != cudaSuccess || !st) return e != cudaSuccess ? ctx_cuda(ctx, e, "ba session") : ctx_fail(ctx, PANO_ERR_CUDA, "ba session: pinned staging allocation failed");
    if (n_pair) memcpy(st, s->table.data(), (size_t)n_pair * sizeof(BaPairDev));
    double* to = (double*)(st + (size_t)n_pair * sizeof(BaPairDev));
    double* fr = to + 2 * nm;
    for (long long i = 0; i < nm; ++i) {
      to[2 * i] = pts[4 * i]; to[2 * i + 1] = pts[4 * i + 1];
      fr[2 * i] = pts[4 * i + 2]; fr[2 * i + 1] = pts[4 * i + 3];
    }
    if (n_pair) e = cudaMemcpyAsync(s->d_pairs, st, (size_t)n_pair * sizeof(BaPairDev), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess && nm) e = cudaMemcpyAsync(s->d_to, to, (size_t)nm * 16, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess && nm) e = cudaMemcpyAsync(s->d_from, fr, (size_t)nm * 16, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) return ctx_cuda(ctx, e, "ba session upload");
  }
  *out = s.release();
  return PANO_OK;
}

extern "C" void pano_ba_session_free(pano_ba_session* s) {
  if (s) ctx_enter(s->ctx);
  delete s;
}

extern "C" int pano_ba_error(pano_ba_session* s, int n_pair, const double* hto_to_from, double* avg, double* max,
                             double* residuals) {
  if (!s) return PANO_ERR_INVALID;
  pano_ctx* ctx = s->ctx;
  ctx_enter(ctx);
  if (n_pair != s->n_pair || (n_pair && !hto_to_from) || !avg || !max)
    return ctx_fail(ctx, PANO_ERR_INVALID, "ba error: %d matrices for a session of %d pairs, or a missing output", n_pair, s->n_pair);
  s->have_error = false;
  const size_t b_res = (size_t)s->nm * 16;
  char* so = nullptr;
  if (residuals && b_res) {                               // before any launch: ctx_pinned2 waits for the stream
    so = (char*)ctx_pinned2(ctx, b_res + 64);
    if (!so) return ctx_fail(ctx, PANO_ERR_CUDA, "ba error: pinned staging allocation failed");
  }
  {
    void* dst[3] = {s->d_hto, s->d_st, s->d_nonfinite};
    const void* src[3] = {hto_to_from, nullptr, nullptr};
    const size_t bytes[3] = {(size_t)n_pair * 72, sizeof(BaErrStats), (size_t)n_pair * 4};
    const int rc = ctx_put_many(ctx, 3, dst, src, bytes);
    if (rc) return rc;
  }
  if (s->nm) {
    dim3 grid((unsigned)std::max(1, std::min((s->max_match + 127) / 128, 1024)), grid_y(n_pair));
    PANO_LAUNCH(ctx, "k_ba_residuals", k_ba_residuals, grid, 128, 0, s->d_pairs, n_pair, s->d_hto, s->d_to, s->d_from, s->d_res,
                s->d_sq, s->d_st, s->d_nonfinite);
  }
  double* h_out = (double*)s->h_out.get();
  PANO_LAUNCH(ctx, "k_ba_error_sum", k_ba_error_sum, 1, 1024, 0, (const float*)s->d_sq, 2 * s->nm, s->d_st, h_out);
  if (so) PANO_CUDA(ctx, cudaMemcpyAsync(so, s->d_res, b_res, cudaMemcpyDeviceToHost, ctx->stream));
  PANO_CUDA(ctx, ctx_spin_stream(ctx));
  *avg = h_out[0];
  *max = h_out[1];
  if (so) memcpy(residuals, so, b_res);
  s->have_error = true;
  return PANO_OK;
}

extern "C" int pano_ba_normal_equations(pano_ba_session* s, int n_pair, const double* mats, double* jtj, double* b,
                                        double* j_rows) {
  if (!s) return PANO_ERR_INVALID;
  pano_ctx* ctx = s->ctx;
  ctx_enter(ctx);
  if (n_pair != s->n_pair || (n_pair && !mats) || !jtj || !b)
    return ctx_fail(ctx, PANO_ERR_INVALID, "ba normal equations: %d pair matrices for a session of %d pairs, or a missing output", n_pair, s->n_pair);
  if (!s->have_error)
    return ctx_fail(ctx, PANO_ERR_INVALID, "ba normal equations: b = J^T r needs the residuals of a pano_ba_error call on this session");
  for (int k = 0; k < n_pair; ++k) memcpy(s->table[k].m, mats + (size_t)k * 117, 117 * sizeof(double));
  const size_t N = (size_t)s->n_cam * 6;
  const size_t b_rows = j_rows ? (size_t)s->nm * 24 * 8 : 0, b_jtj = N * N * 8, b_b = N * 8;
  char* so = (char*)ctx_pinned2(ctx, b_rows + b_jtj + b_b + 64);
  if (!so) return ctx_fail(ctx, PANO_ERR_CUDA, "ba normal equations: pinned staging allocation failed");
  if (n_pair) {
    const int rc = ctx_put(ctx, s->d_pairs, s->table.data(), (size_t)n_pair * sizeof(BaPairDev));
    if (rc) return rc;
  }
  if (n_pair && s->max_match) {
    dim3 grid((unsigned)std::max(1, std::min((s->max_match + 127) / 128, 1024)), grid_y(n_pair));
    PANO_LAUNCH(ctx, "k_ba_rows", k_ba_rows, grid, 128, 0, (const BaPairDev*)s->d_pairs, n_pair, (const double2*)s->d_to,
                s->d_rows);
  }
  PANO_LAUNCH(ctx, "k_ba_jtj", k_ba_jtj, dim3((unsigned)s->n_cam, (unsigned)s->n_cam), 64, 0, (const BaPairDev*)s->d_pairs,
              n_pair, s->n_cam, (const double*)s->d_rows, s->d_jtj);
  PANO_LAUNCH(ctx, "k_ba_jtr", k_ba_jtr, (unsigned)N, 128, 0, (const BaPairDev*)s->d_pairs, n_pair, (const double*)s->d_rows,
              (const double*)s->d_res, (const int*)s->d_nonfinite, s->d_b);
  if (b_rows) PANO_CUDA(ctx, cudaMemcpyAsync(so, s->d_rows, b_rows, cudaMemcpyDeviceToHost, ctx->stream));
  PANO_CUDA(ctx, cudaMemcpyAsync(so + b_rows, s->d_jtj, b_jtj, cudaMemcpyDeviceToHost, ctx->stream));
  PANO_CUDA(ctx, cudaMemcpyAsync(so + b_rows + b_jtj, s->d_b, b_b, cudaMemcpyDeviceToHost, ctx->stream));
  PANO_CUDA(ctx, ctx_spin_stream(ctx));
  if (b_rows) memcpy(j_rows, so, b_rows);
  memcpy(jtj, so + b_rows, b_jtj);
  memcpy(b, so + b_rows + b_jtj, b_b);
  return PANO_OK;
}
