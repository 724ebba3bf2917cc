// Unique log-uniform candidate sampler of the sampled-softmax training step (c2v_sample_log_uniform, include/c2v_b200.h):
// tf.random.log_uniform_candidate_sampler(unique=True) -- TF's LogUniformSampler / RangeSampler::SampleBatchGetExpectedCount
// -- on its own Philox stream.  One CTA draws in rounds of kSamplerThreads draws, in draw order: every draw stamps its
// value's slot of a per-class table with (call tag, draw index) by atomicMin, so after the round a draw is the first
// occurrence of its value exactly when the slot still holds its own index; a block scan of those flags gives every first
// occurrence its rank among all first occurrences so far.  The first S of them in draw order are the sample, and the
// draw that supplied the S-th is num_tries -- the sequential definition, whatever order the atomics land in.
// tests/sampler_model.py states the definition; tests/test_gpu_sampled_training.py holds the kernel to it.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "common.cuh"

namespace c2v {

namespace {

constexpr int kSamplerThreads = 1024;                  // draws per round
constexpr int64_t kSamplerMaxDraws = int64_t(1) << 31; // draw cap; a multiple of kSamplerThreads
constexpr int kSamplerMaxS = 1024;

// uniform double in [0, 1) from the 53 top bits of words x (27 bits) and y (26 bits) of Philox4x32-10 at counter
// (i, 0, step_lo, step_hi)
__device__ __forceinline__ double sampler_uniform(uint32_t i, uint2 step, uint2 key) {
  const uint4 r = philox4x32_10(make_uint4(i, 0u, step.x, step.y), key);
  return (double)((uint64_t)(r.x >> 5) * 67108864ull + (uint64_t)(r.y >> 6)) * 0x1p-53;
}

// log of the expected count of class c in num_tries draws (TF's ExpectedCountHelper, in double), rounded once to float
__device__ __forceinline__ float sampler_logq(int32_t c, double log_range, int S, int64_t tries) {
  const double p = log(((double)c + 2.0) / ((double)c + 1.0)) / log_range;
  const double count = (tries == (int64_t)S) ? (double)S * p : -expm1((double)tries * log1p(-p));
  return (float)log(count);
}

__global__ void __launch_bounds__(kSamplerThreads, 1)
log_uniform_sample_kernel(int32_t Y, double log_range, int32_t S, const int32_t* __restrict__ target, int32_t B,
                          uint2 key, uint2 step, uint32_t tag, unsigned long long* __restrict__ stamp,
                          int32_t* __restrict__ sampled, float* __restrict__ logq_true, float* __restrict__ logq_sampled,
                          int64_t* __restrict__ num_tries, int32_t* __restrict__ cap_hits) {
  __shared__ int32_t s_val[kSamplerMaxS];
  __shared__ int32_t s_warp[kSamplerThreads / kWarp];
  __shared__ long long s_tries;
  const int tid = threadIdx.x, lane = tid & (kWarp - 1), warp = tid >> 5;
  if (tid == 0) s_tries = 0;
  int found = 0;                                       // first occurrences so far (uniform over the block)
  for (int64_t base = 0; base < kSamplerMaxDraws && found < S; base += kSamplerThreads) {
    const uint32_t i = (uint32_t)(base + tid);
    const double u = sampler_uniform(i, step, key);
    const int64_t v = ((int64_t)floor(exp(u * log_range)) - 1) % (int64_t)Y;
    const unsigned long long mine = ((unsigned long long)tag << 32) | i;
    atomicMin(stamp + v, mine);
    __syncthreads();                                   // every draw of the round has stamped its value
    const bool first = __ldcg(stamp + v) == mine;
    const unsigned ballot = __ballot_sync(0xffffffffu, first);
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll 8
    for (int w = 0; w < kSamplerThreads / kWarp; ++w) {
      const int n = s_warp[w];
      before += w < warp ? n : 0;
      total += n;
    }
    if (first) {
      const int pos = found + before + __popc(ballot & ((1u << lane) - 1u));
      if (pos < S) {
        s_val[pos] = (int32_t)v;
        if (pos == S - 1) s_tries = (long long)i + 1;
      }
    }
    found += total;
    __syncthreads();                                   // s_warp is rewritten by the next round
  }
  if (found < S) {                                     // the cap was reached: flag it, fill the rest with class 0
    for (int s = found + tid; s < S; s += kSamplerThreads) s_val[s] = 0;
    if (tid == 0) {
      s_tries = kSamplerMaxDraws;
      atomicAdd(cap_hits, 1);
    }
  }
  __syncthreads();
  const int64_t tries = s_tries;
  for (int s = tid; s < S; s += kSamplerThreads) {
    const int32_t c = s_val[s];
    sampled[s] = c;
    logq_sampled[s] = sampler_logq(c, log_range, S, tries);
  }
  for (int b = tid; b < B; b += kSamplerThreads) logq_true[b] = sampler_logq(__ldg(target + b), log_range, S, tries);
  if (tid == 0 && num_tries) *num_tries = tries;
}

}  // namespace

// Launches the sampler of c2v_sample_log_uniform (arguments checked by the caller; stamp: [Y] slots whose tags are all
// below `tag`'s, e.g. all ones before the first call and tags counting down from 0xFFFFFFFE).
cudaError_t launch_log_uniform_sampler(int32_t Y, double log_range, int32_t S, const int32_t* target, int32_t B,
                                       uint64_t seed, uint64_t step, uint32_t tag, unsigned long long* stamp,
                                       int32_t* sampled, float* logq_true, float* logq_sampled, int64_t* num_tries,
                                       int32_t* cap_hits, cudaStream_t st) {
  // the dropout mask's key is (seed_lo, seed_hi); the sampler's differs from it in both words for every seed
  const uint2 key = make_uint2((uint32_t)seed ^ 0x6C6F6775u, (uint32_t)(seed >> 32) ^ 0x73616D70u);
  const uint2 stp = make_uint2((uint32_t)step, (uint32_t)(step >> 32));
  log_uniform_sample_kernel<<<1, kSamplerThreads, 0, st>>>(Y, log_range, S, target, B, key, stp, tag, stamp, sampled,
                                                            logq_true, logq_sampled, num_tries, cap_hits);
  return cudaGetLastError();
}

}  // namespace c2v
