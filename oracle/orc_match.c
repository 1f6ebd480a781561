/*
 * orc_match.c — plain-C restatement of the reference's exact matcher.
 * TEST INFRASTRUCTURE ONLY (see orc_common.h).  Citations relative to
 * the reference's src/.
 */
#include <float.h>
#include "orc_common.h"

/* feature/dist.cc:22-57, the SSE branch (what -march=native / -msse3 builds of
 * the reference execute): four independent lane accumulators over the 32
 * 4-float steps, lane sum (l0+l1)+(l2+l3) (two _mm_hadd_ps).  The early exit
 * (partial sum > now_thres, checked at n = 128, 96, 64, 32 remaining) returns
 * FLT_MAX; it never changes a decision because partial sums are monotone. */
static float euclidean_sqr(const float* x, const float* y, int n, float now_thres) {
  float l0 = 0, l1 = 0, l2 = 0, l3 = 0;
  for (; n > 0; n -= 4) {
    float d0 = x[0] - y[0], d1 = x[1] - y[1], d2 = x[2] - y[2], d3 = x[3] - y[3];
    l0 = l0 + d0 * d0; l1 = l1 + d1 * d1; l2 = l2 + d2 * d2; l3 = l3 + d3 * d3;
    if (n % 32 == 0) {
      float ans = (l0 + l1) + (l2 + l3);
      if (ans > now_thres) return FLT_MAX;
    }
    x += 4; y += 4;
  }
  return (l0 + l1) + (l2 + l3);
}

/* feature/matcher.cc:15-71 FeatureMatcher::match.  The decision of row k depends on
 * nothing but k, so the loop body is written as "decide row k -> idx[k]" followed by
 * the single-thread emission order (ascending k); the ORC_MT build (liboracle_mt.so,
 * a faster checker for the BASELINE-size configs) runs the rows on all host threads. */
int orc_match(const float* a, int n, const float* b, int m, const pano_params* P,
              int* pairs, int* npairs) {
  const float REJECT_RATIO_SQR = P->match_reject_next_ratio * P->match_reject_next_ratio;
  int l1 = n, l2 = m, rev = l1 > l2, k, cnt = 0;
  const float *f1 = a, *f2 = b;
  int* idx;
  if (rev) { l1 = m; l2 = n; f1 = b; f2 = a; }
  idx = (int*)malloc(sizeof(int) * (size_t)(l1 > 0 ? l1 : 1));
  ORC_PAR_FOR(schedule(dynamic, 16))
  for (k = 0; k < l1; ++k) {
    const float* dsc1 = f1 + (size_t)128 * k;
    const float* dsc2;
    int min_idx = -1, kk;
    float mn = FLT_MAX, next_min = FLT_MAX;
    idx[k] = -1;
    for (kk = 0; kk < l2; ++kk) {
      float dist = euclidean_sqr(dsc1, f2 + (size_t)128 * kk, 128, next_min);
      if (dist < mn) { next_min = mn; mn = dist; min_idx = kk; }
      else if (dist < next_min) next_min = dist;
    }
    if (mn > REJECT_RATIO_SQR * next_min) continue;
    dsc2 = f2 + (size_t)128 * min_idx;
    for (kk = 0; kk < l1; ++kk)
      if (kk != k) {
        float dist = euclidean_sqr(dsc2, f1 + (size_t)128 * kk, 128, next_min);
        if (dist < next_min) next_min = dist;
      }
    if (mn > REJECT_RATIO_SQR * next_min) continue;
    idx[k] = min_idx;
  }
  for (k = 0; k < l1; ++k) {
    if (idx[k] < 0) continue;
    if (rev) { pairs[2 * cnt] = idx[k]; pairs[2 * cnt + 1] = k; }
    else { pairs[2 * cnt] = k; pairs[2 * cnt + 1] = idx[k]; }
    ++cnt;
  }
  free(idx);
  *npairs = cnt;
  return 0;
}
