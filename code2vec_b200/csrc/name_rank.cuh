// Scores of each example's own name over the whole target vocabulary (c2v_name_scores, DESIGN.md §6n), from the logits
// slab S[b, 0:Y] the logits GEMM left (pitch ldS, the row c2v_topk scans).
#pragma once
#include <limits.h>
#include "common.cuh"

namespace c2v {

// One CTA per row; at 512 threads a java14m row (261,245 logits) is 128 float4s per thread
constexpr int kNameRankThreads = 512;
constexpr int kNameRankWarps = kNameRankThreads / 32;

// (max, lowest index of the max, sum exp(x - max)) of two disjoint parts of a row; -inf max = an empty part.  Symmetric in
// its two arguments (the sum's two products are added in either order to the same float), so both lanes of a butterfly
// step hold the same result.
__device__ __forceinline__ void name_rank_fold(float& m, float& s, int& i, float om, float os, int oi) {
  const float M = fmaxf(m, om);
  const float a = (m > -INFINITY) ? s * expf(m - M) : 0.f;
  const float c = (om > -INFINITY) ? os * expf(om - M) : 0.f;
  if (om > m || (om == m && oi < i)) i = oi;
  m = M;
  s = a + c;
}

// For row b with target y = target[b] and t = S[b, y]:
//   rank[b]      = 1 + #{j : S[j] > t} + #{j < y : S[j] == t}       (tf.nn.top_k's order, as topk_kernel ranks the row)
//   logp[b]      = t - lse, lse = m + log sum_j exp(S[j] - m), m = max_j S[j]  (computed as (t - m) - log sum)
//   top1[b]      = the lowest j with S[j] == m                         (topk_kernel's first id)
//   top1_logp[b] = m - lse                                             (computed as -log sum)
// A row holding a NaN: rank 0 and NaN log-probabilities (top1 still the lowest index of the largest non-NaN logit).  A
// target outside [0, Y): rank -1 and NaN log-probabilities.  One pass: t first, then each thread walks its float4s in
// increasing column order keeping its counts, its (max, first argmax) and an online sum exp; warp shuffles, then shared
// memory, combine them.  The counts are integers, so no summation order changes them.
__global__ void __launch_bounds__(kNameRankThreads)
name_rank_kernel(const float* __restrict__ S, size_t ldS, int Y, const int32_t* __restrict__ target, int32_t* __restrict__ rank,
                 float* __restrict__ logp, int32_t* __restrict__ top1, float* __restrict__ top1_logp) {
  __shared__ float red_m[kNameRankWarps], red_s[kNameRankWarps];
  __shared__ int red_i[kNameRankWarps], red_gt[kNameRankWarps], red_eq[kNameRankWarps], red_nan[kNameRankWarps];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* row = S + (size_t)b * ldS;
  const int y = target[b];
  const bool valid = y >= 0 && y < Y;
  const float t = valid ? row[y] : __int_as_float(0x7fffffff);   // NaN: no comparison with it holds
  int gt = 0, eq = 0, nan = 0;
  float m = -INFINITY, s = 0.f;
  int i = INT_MAX;
  auto count = [&](float x, int j) {
    nan |= (x != x);
    gt += (x > t);
    eq += (x == t) & (j < y);
  };
  auto take4 = [&](const float4 x, int j) {
    count(x.x, j); count(x.y, j + 1); count(x.z, j + 2); count(x.w, j + 3);
    const float m4 = fmaxf(fmaxf(x.x, x.y), fmaxf(x.z, x.w));
    if (m4 > m) {                       // a strictly larger max: earlier columns of this thread keep no claim to it
      s *= expf(m - m4);
      m = m4;
      i = j + (x.x == m4 ? 0 : x.y == m4 ? 1 : x.z == m4 ? 2 : 3);
    }
    if (m > -INFINITY) s += expf(x.x - m) + expf(x.y - m) + expf(x.z - m) + expf(x.w - m);
  };
  // kNameRankLoads float4s in flight per thread: all loads of a round are issued before any of them is used
  constexpr int kNameRankLoads = 4;
  const int Y4 = Y >> 2;
  for (int q0 = tid; q0 < Y4; q0 += kNameRankLoads * kNameRankThreads) {
    float4 x[kNameRankLoads];
#pragma unroll
    for (int u = 0; u < kNameRankLoads; ++u) {
      const int q = q0 + u * kNameRankThreads;
      if (q < Y4) x[u] = *reinterpret_cast<const float4*>(row + 4 * q);
    }
#pragma unroll
    for (int u = 0; u < kNameRankLoads; ++u) {
      const int q = q0 + u * kNameRankThreads;
      if (q < Y4) take4(x[u], 4 * q);
    }
  }
  for (int j = 4 * Y4 + tid; j < Y; j += kNameRankThreads) {
    const float x = row[j];
    count(x, j);
    if (x > m) { s *= expf(m - x); m = x; i = j; }
    if (m > -INFINITY) s += expf(x - m);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    name_rank_fold(m, s, i, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o),
                   __shfl_xor_sync(0xffffffffu, i, o));
  gt = __reduce_add_sync(0xffffffffu, gt);
  eq = __reduce_add_sync(0xffffffffu, eq);
  nan = __reduce_or_sync(0xffffffffu, nan);
  if (lane == 0) {
    red_m[warp] = m; red_s[warp] = s; red_i[warp] = i;
    red_gt[warp] = gt; red_eq[warp] = eq; red_nan[warp] = nan;
  }
  __syncthreads();
  if (tid != 0) return;
  for (int w = 1; w < kNameRankWarps; ++w) {
    name_rank_fold(m, s, i, red_m[w], red_s[w], red_i[w]);
    gt += red_gt[w];
    eq += red_eq[w];
    nan |= red_nan[w];
  }
  const float ls = logf(s);
  const bool scored = valid && !nan;
  rank[b] = !valid ? -1 : nan ? 0 : 1 + gt + eq;
  logp[b] = scored ? (t - m) - ls : __int_as_float(0x7fffffff);
  top1[b] = i;
  top1_logp[b] = scored ? -ls : __int_as_float(0x7fffffff);
}

}  // namespace c2v
