// Shared device helpers for the path-attention engine (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

namespace c2v {

constexpr int kWarp = 32;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---------------------------------------------------------------------------------------------
// theta <- theta - (lr_t m) / (sqrt(v) + eps): the parameter move of TF1 Adam in correctly rounded fp32 operations, shared by
// every kernel that applies it (adam_kernel, the lazy row replay, the dY epilogue) so that they stay bit-identical.
// tests/adam_model.py states the step; tests/test_gpu_adam_model.py holds every path to it bit for bit.
// A ZERO numerator -- an element whose gradient has been exactly zero so far (dropout masks a quarter of every row; rows
// no batch has touched), or lr_t m underflowing -- makes the correctly rounded quotient a zero of the numerator's sign
// when the denominator is positive, so theta - num is the same bits as theta - num / den.  Dividing anyway sends div.rn.f32
// through its out-of-line slow path (zero / denormal operands), which a profile of the row replay showed on 46 % of the
// divisions of a 25-step run; the branch keeps it for genuinely denormal numerators only.  The denominator is positive
// for every v >= 0 only when eps > 0 (pos_eps, decided by the caller from the step's eps): with eps = 0 an element with
// m = v = 0 divides 0 / 0 into NaN, and a negative eps can flip the zero's sign, exactly as the dense kernel does.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float adam_move(float theta, float lr_t, float m, float v, float eps, bool pos_eps) {
  const float num = __fmul_rn(lr_t, m);
  if (pos_eps && num == 0.f) return __fsub_rn(theta, num);
  return __fsub_rn(theta, __fdiv_rn(num, __fadd_rn(__fsqrt_rn(v), eps)));
}
// exp_slab schedule (umma::EpiExpSumT, expsum_combine_kernel): a row's largest U = exp(logit - c_row) must stay inside this
// window for the deferred normalisation to be used; fp32 then still resolves elements e^-27 below the row's maximum and
// a sum of 2^18 such terms cannot overflow.  Its factor r = 1 / (B Z) must also leave dY's operand r v_b normal where it
// matters: r max_j |v_b[j]| >= kExpSlabMinOperand, 2^14 above FLT_MIN.  A subnormal operand loses the 13 bits the tf32
// tensor cores (and each half of the 3xTF32 split) drop from the bottom of its field, 2^-136 absolutely; above this
// limit that is below 2^-24 of the row's largest operand.  Z reaches 2.6e35 inside the U window (Y = 261,246), where r
// falls below FLT_MIN at B = 1024.
constexpr float kExpSlabMin = 1e-26f, kExpSlabMax = 1e30f;
constexpr float kExpSlabMinOperand = 0x1p-112f;

// The same move without the test, for dense gradients (the target table's update in the dY epilogue, adam_kernel): zero
// numerators are rare there and the branch costs more than the occasional slow path.  Identical bits to adam_move, for
// every eps, by the argument above.
__device__ __forceinline__ float adam_move_dense(float theta, float lr_t, float m, float v, float eps) {
  return __fsub_rn(theta, __fdiv_rn(__fmul_rn(lr_t, m), __fadd_rn(__fsqrt_rn(v), eps)));
}

// ---------------------------------------------------------------------------------------------
// 3xTF32 operand split (C2V_MATH_3XTF32): x = hi + lo + O(2^-22 |x|) with hi, lo representable in tf32
// (10 explicit mantissa bits), both rounded to nearest so the tensor core's own handling of the low
// 13 bits of a 32-bit operand never matters.  A fp32 product a.b is then issued as
// a_lo.b_hi + a_hi.b_lo + a_hi.b_hi with fp32 accumulation; the dropped a_lo.b_lo term is O(2^-22 |a b|).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = tf32_rna(x);
  lo = tf32_rna(x - hi);
}
__device__ __forceinline__ void split_tf32(const float4& x, float4& hi, float4& lo) {
  split_tf32(x.x, hi.x, lo.x); split_tf32(x.y, hi.y, lo.y); split_tf32(x.z, hi.z, lo.z); split_tf32(x.w, hi.w, lo.w);
}

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., SC'11).  Counter-based, so the dropout mask of the forward pass
// is regenerated -- not stored -- in the backward pass, and oracle/path_attention_oracle.py
// (dropout_keep_mask) reproduces it bit for bit.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
    const uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += W0;
    k.y += W1;
  }
  return c;
}

// Dropout description shared by the forward and backward kernels.
//   ext   : caller-supplied 0/1 mask [rows, ctx_dim] (tests) or nullptr
//   thr   : keep iff u32 < thr   (thr = floor(keep * 2^32)); enabled == 0 -> identity
//   scale : 1/keep, applied to survivors   (tensorflow_model.py:245-246: x * scale * mask)
struct Dropout {
  const float* ext;
  uint32_t thr;
  float scale;
  uint2 key;      // (seed_lo, seed_hi)
  uint2 step;     // (step_lo, step_hi)
  int ctx_dim;    // 3d
  int enabled;
};

// Multipliers (0 or scale) for the 4 consecutive columns [col4*4, col4*4+4) of context row `row`.
__device__ __forceinline__ float4 dropout_mult4(const Dropout& dp, int row, int col4) {
  if (!dp.enabled) return make_float4(1.f, 1.f, 1.f, 1.f);
  if (dp.ext) {
    const float4 m = *reinterpret_cast<const float4*>(dp.ext + (size_t)row * dp.ctx_dim + col4 * 4);
    return make_float4(m.x * dp.scale, m.y * dp.scale, m.z * dp.scale, m.w * dp.scale);
  }
  const uint4 r = philox4x32_10(make_uint4((uint32_t)row, (uint32_t)col4, dp.step.x, dp.step.y), dp.key);
  return make_float4(r.x < dp.thr ? dp.scale : 0.f, r.y < dp.thr ? dp.scale : 0.f,
                     r.z < dp.thr ? dp.scale : 0.f, r.w < dp.thr ? dp.scale : 0.f);
}

// An embedding table that may be row-sharded over up to 8 GPUs of one NVSwitch domain: global row
// r lives on shard (r & mask) at local row (r >> shift); base[] holds the local shard and the
// peers' shards mapped through CUDA IPC, so gathers are plain loads and gradient scatter-adds are
// plain red.global.add over NVLink.  A replicated / single-GPU table is the 1-shard case.
constexpr int kMaxShards = 8;
struct ShardedTable {
  float* base[kMaxShards];
  int shift;
  int mask;
};
__device__ __forceinline__ float* table_row(const ShardedTable& t, int idx, int d) {
  return t.base[idx & t.mask] + (size_t)(idx >> t.shift) * d;
}

// The three index arrays + two tables that define the gathered context matrix
// X[n, 0:3d] = [ tok[src[n]] | path[pth[n]] | tok[tgt[n]] ]      (tensorflow_model.py:238-243)
struct ContextSource {
  const int32_t* src;
  const int32_t* pth;
  const int32_t* tgt;
  ShardedTable tok;     // [T, d]
  ShardedTable path;    // [P, d]
  int d;
  int rows;             // B*C
};

// pointer to X[n, j] for j in segment-aligned groups of 4 (d % 4 == 0 so a float4 never straddles)
__device__ __forceinline__ const float* ctx_ptr(const ContextSource& cs, int n, int j) {
  const int seg = j / cs.d;
  const int off = j - seg * cs.d;
  if (seg == 0) return table_row(cs.tok, __ldg(cs.src + n), cs.d) + off;
  if (seg == 1) return table_row(cs.path, __ldg(cs.pth + n), cs.d) + off;
  return table_row(cs.tok, __ldg(cs.tgt + n), cs.d) + off;
}

}  // namespace c2v
