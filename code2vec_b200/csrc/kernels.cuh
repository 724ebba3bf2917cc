// Non-GEMM kernels of the path-attention engine: attention softmax / weighted sum and its
// backward, fused cross-entropy, top-k, TF1 Adam, small deterministic reductions.
#pragma once
#include <float.h>
#include <limits.h>
#include "common.cuh"

namespace c2v {

// one CTA per example: 128 threads and <= 64 registers make 8 CTAs resident per SM, so a 1024-example batch is ONE wave on
// the H100's 132 SMs (1056 slots)
constexpr int kAttnThreads = 128;
constexpr int kAttnWarps = kAttnThreads / 32;

// Deterministic block-wide sum (fixed tree); `red` is shared scratch of >= 32 floats.
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f;
  if (warp == 0) {
    r = warp_sum(r);
    if (lane == 0) red[0] = r;
  }
  __syncthreads();
  r = red[0];
  __syncthreads();
  return r;
}
__device__ __forceinline__ float block_max(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = (threadIdx.x < nw) ? red[threadIdx.x] : -INFINITY;
  if (warp == 0) {
    r = warp_max(r);
    if (lane == 0) red[0] = r;
  }
  __syncthreads();
  r = red[0];
  __syncthreads();
  return r;
}

// ---------------------------------------------------------------------------------------------
// Attention forward: z_c = h_c . a + log(mask_c); alpha = softmax_c(z); v = sum_c alpha_c h_c
// (tensorflow_model.py:254-263).  One CTA per example (bag); a warp per context; online softmax
// so H is read once.  A bag with no valid context gives NaN (tf.nn.softmax of all -inf).
// ---------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(kAttnThreads, NV <= 3 ? 8 : 4)
attn_fwd_kernel(const float* __restrict__ H, const float* __restrict__ a, const float* __restrict__ mask,
                int C, int D, float* __restrict__ alpha, float* __restrict__ v) {
  extern __shared__ float sm[];
  float* zs = sm;                       // [C]
  float* red = zs + ((C + 3) & ~3);     // [32]
  float* wm = red + 32;                 // [kAttnWarps]
  float* vbuf = wm + kAttnWarps;        // [kAttnWarps][D]
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  float4 av[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int j = i * 128 + lane * 4;
    av[i] = (j < D) ? *reinterpret_cast<const float4*>(a + j) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float m_w = -INFINITY;
  float4 acc[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);

  for (int c = warp; c < C; c += kAttnWarps) {
    const float* h = H + ((size_t)b * C + c) * D;
    float4 hv[NV];
    float part = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int j = i * 128 + lane * 4;
      hv[i] = (j < D) ? *reinterpret_cast<const float4*>(h + j) : make_float4(0.f, 0.f, 0.f, 0.f);
      part += hv[i].x * av[i].x + hv[i].y * av[i].y + hv[i].z * av[i].z + hv[i].w * av[i].w;
    }
    const float z = warp_sum(part) + logf(mask[(size_t)b * C + c]);     // log(0) = -inf
    if (lane == 0) zs[c] = z;
    const float nm = fmaxf(m_w, z);
    if (nm > -INFINITY) {                        // NaN z falls through: poisons acc like TF would
      const float sc = expf(m_w - nm), e = expf(z - nm);
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        acc[i].x = acc[i].x * sc + e * hv[i].x;
        acc[i].y = acc[i].y * sc + e * hv[i].y;
        acc[i].z = acc[i].z * sc + e * hv[i].z;
        acc[i].w = acc[i].w * sc + e * hv[i].w;
      }
      m_w = nm;
    } else if (z != z) {
      m_w = z;
    }
  }
  if (lane == 0) wm[warp] = m_w;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int j = i * 128 + lane * 4;
    if (j < D) *reinterpret_cast<float4*>(vbuf + (size_t)warp * D + j) = acc[i];
  }
  __syncthreads();
  float zmax = -INFINITY;
  for (int c = tid; c < C; c += kAttnThreads) zmax = fmaxf(zmax, zs[c]);
  zmax = block_max(zmax, red);
  float s = 0.f;
  for (int c = tid; c < C; c += kAttnThreads) s += expf(zs[c] - zmax);    // -inf - -inf = NaN: all-masked bag
  s = block_sum(s, red);
  const float inv = 1.f / s;
  if (alpha)
    for (int c = tid; c < C; c += kAttnThreads) alpha[(size_t)b * C + c] = expf(zs[c] - zmax) * inv;
  for (int j = tid; j < D; j += kAttnThreads) {
    float r = 0.f;
#pragma unroll
    for (int w = 0; w < kAttnWarps; ++w) {
      const float mw = wm[w];
      if (mw > -INFINITY || mw != mw) r += vbuf[(size_t)w * D + j] * expf(mw - zmax);
    }
    v[(size_t)b * D + j] = (zmax > -INFINITY) ? r * inv : NAN;
  }
}

// ---------------------------------------------------------------------------------------------
// Attention backward (SURVEY A.2):  dalpha_c = h_c . dv ; dz_c = alpha_c (dalpha_c - t), t = sum_c alpha_c dalpha_c ;
// dh = alpha dv + dz a ; du = dh (1 - h^2) written over H ; da partial per example.
// t needs no pass of its own: sum_c alpha_c (h_c . dv) = (sum_c alpha_c h_c) . dv = v . dv with the code vector v the
// forward pass already produced -- so H is read ONCE and overwritten in the same pass (a warp per context: the dot
// product, dz and du all come from the row the warp holds in registers).
// ---------------------------------------------------------------------------------------------
// NV <= 3 (D <= 384): 8 resident CTAs per SM (64 registers) hold a 1024-example batch in one wave on 132 SMs; 7 would
// leave a second wave, which costs more than the few spilled registers
template <int NV, bool SPLIT>
__global__ void __launch_bounds__(kAttnThreads, NV <= 3 ? 8 : 4)
attn_bwd_kernel(float* __restrict__ H, const float* __restrict__ alpha, const float* __restrict__ dv,
                const float* __restrict__ v, const float* __restrict__ a, int C, int D, float* __restrict__ da_part,
                float* __restrict__ H_lo) {
  // SPLIT (3xTF32): dU is written as its tf32 split, high parts over H and residuals into H_lo
  extern __shared__ float sm[];
  float* dabuf = sm;                    // [kAttnWarps][D]
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float4 av[NV], gv[NV], dacc[NV];
  float tp = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int j = i * 128 + lane * 4;
    const bool ok = j < D;
    av[i] = ok ? *reinterpret_cast<const float4*>(a + j) : make_float4(0.f, 0.f, 0.f, 0.f);
    gv[i] = ok ? *reinterpret_cast<const float4*>(dv + (size_t)b * D + j) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 vv = ok ? *reinterpret_cast<const float4*>(v + (size_t)b * D + j) : make_float4(0.f, 0.f, 0.f, 0.f);
    tp += vv.x * gv[i].x + vv.y * gv[i].y + vv.z * gv[i].z + vv.w * gv[i].w;
    dacc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const float t = warp_sum(tp);         // the same value, bit for bit, in every warp of the CTA
  for (int c = warp; c < C; c += kAttnWarps) {
    const float al = alpha[(size_t)b * C + c];
    float* h = H + ((size_t)b * C + c) * D;
    if (al == 0.f) {                    // masked context: exact zeros (alpha == 0)
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int j = i * 128 + lane * 4;
        if (j < D) {
          *reinterpret_cast<float4*>(h + j) = make_float4(0.f, 0.f, 0.f, 0.f);
          if (SPLIT) *reinterpret_cast<float4*>(H_lo + ((size_t)b * C + c) * D + j) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
      continue;
    }
    float4 hv[NV];
    float part = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int j = i * 128 + lane * 4;
      hv[i] = (j < D) ? *reinterpret_cast<const float4*>(h + j) : make_float4(0.f, 0.f, 0.f, 0.f);
      part += hv[i].x * gv[i].x + hv[i].y * gv[i].y + hv[i].z * gv[i].z + hv[i].w * gv[i].w;
    }
    const float dz = al * (warp_sum(part) - t);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int j = i * 128 + lane * 4;
      if (j < D) {
        float4 du;
        du.x = (al * gv[i].x + dz * av[i].x) * (1.f - hv[i].x * hv[i].x);
        du.y = (al * gv[i].y + dz * av[i].y) * (1.f - hv[i].y * hv[i].y);
        du.z = (al * gv[i].z + dz * av[i].z) * (1.f - hv[i].z * hv[i].z);
        du.w = (al * gv[i].w + dz * av[i].w) * (1.f - hv[i].w * hv[i].w);
        if (SPLIT) {
          float4 hi, lo;
          split_tf32(du, hi, lo);
          *reinterpret_cast<float4*>(h + j) = hi;
          *reinterpret_cast<float4*>(H_lo + ((size_t)b * C + c) * D + j) = lo;
        } else {
          *reinterpret_cast<float4*>(h + j) = du;
        }
        dacc[i].x += dz * hv[i].x; dacc[i].y += dz * hv[i].y; dacc[i].z += dz * hv[i].z; dacc[i].w += dz * hv[i].w;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int j = i * 128 + lane * 4;
    if (j < D) *reinterpret_cast<float4*>(dabuf + (size_t)warp * D + j) = dacc[i];
  }
  __syncthreads();
  for (int j = tid; j < D; j += kAttnThreads) {
    float r = 0.f;
#pragma unroll
    for (int w = 0; w < kAttnWarps; ++w) r += dabuf[(size_t)w * D + j];
    da_part[(size_t)b * D + j] = r;
  }
}

// ---------------------------------------------------------------------------------------------
// Fused sparse-softmax cross entropy over one row of the logits slab S[b, 0:Y]
// (tensorflow_model.py:227-230).  Pass 1: online (max, sum-exp) -> lse, loss_b = lse - S[y_b].
// Pass 2 (write_probs): S <- (softmax - onehot) / B in place  = dL/dlogits.
// ---------------------------------------------------------------------------------------------
constexpr int kXentThreads = 512;

__global__ void __launch_bounds__(kXentThreads)
xent_kernel(float* __restrict__ S, size_t ldS, const int32_t* __restrict__ target, int Y, float inv_batch,
            float* __restrict__ loss_b, float* __restrict__ lse_out, int write_probs) {
  __shared__ float red[32];
  float* row = S + (size_t)blockIdx.x * ldS;
  const int tid = threadIdx.x;
  const int Y4 = Y >> 2;
  const int y = target[blockIdx.x];
  const float logit_y = row[y];          // read before pass 2 overwrites the row
  float m = -INFINITY, s = 0.f;
  for (int q = tid; q < Y4; q += kXentThreads) {
    const float4 x = *reinterpret_cast<const float4*>(row + 4 * q);
    const float m4 = fmaxf(fmaxf(x.x, x.y), fmaxf(x.z, x.w));
    if (m4 > m) { s *= expf(m - m4); m = m4; }
    s += expf(x.x - m) + expf(x.y - m) + expf(x.z - m) + expf(x.w - m);
  }
  for (int j = 4 * Y4 + tid; j < Y; j += kXentThreads) {
    const float x = row[j];
    if (x > m) { s *= expf(m - x); m = x; }
    s += expf(x - m);
  }
  const float M = block_max(m, red);
  s = (m > -INFINITY) ? s * expf(m - M) : 0.f;
  s = block_sum(s, red);
  const float lse = M + logf(s);
  if (tid == 0) {
    loss_b[blockIdx.x] = lse - logit_y;
    if (lse_out) lse_out[blockIdx.x] = lse;
  }
  if (!write_probs) return;
  for (int q = tid; q < Y4; q += kXentThreads) {
    float4 x = *reinterpret_cast<const float4*>(row + 4 * q);
    x.x = expf(x.x - lse) * inv_batch; x.y = expf(x.y - lse) * inv_batch;
    x.z = expf(x.z - lse) * inv_batch; x.w = expf(x.w - lse) * inv_batch;
    const int j = 4 * q;
    if (y >= j && y < j + 4) {
      if (y == j) x.x -= inv_batch; else if (y == j + 1) x.y -= inv_batch;
      else if (y == j + 2) x.z -= inv_batch; else x.w -= inv_batch;
    }
    *reinterpret_cast<float4*>(row + 4 * q) = x;
  }
  for (int j = 4 * Y4 + tid; j < (int)ldS; j += kXentThreads) {
    float p = 0.f;
    if (j < Y) { p = expf(row[j] - lse) * inv_batch; if (j == y) p -= inv_batch; }
    row[j] = p;                          // padding columns [Y, ldS) are zeroed
  }
}

// tf32 path: the logits GEMM epilogue already produced per-(row, n-tile) (max, sum exp) partials.
// xent_combine_kernel: lse_b from the partials, loss_b = lse_b - S[b, y_b].   One CTA per row.
__global__ void __launch_bounds__(256)
xent_combine_kernel(const float2* __restrict__ partial, int n_tiles, const float* __restrict__ S, size_t ldS,
                    const int32_t* __restrict__ target, float* __restrict__ loss_b, float* __restrict__ lse_out,
                    const float* __restrict__ true_logit = nullptr, const int* __restrict__ gate = nullptr,
                    float* __restrict__ rscale_one = nullptr, unsigned* __restrict__ gate_count = nullptr) {
  // gate: this launch is the fallback of the exp_slab schedule and does nothing while *gate == 0; when it runs, the rows'
  // deferred factors become 1 (the slab will hold the finished gradient) and the fallback counter moves
  if (gate && *gate == 0) return;
  __shared__ float red[32];
  const int b = blockIdx.x;
  if (rscale_one && threadIdx.x == 0) rscale_one[b] = 1.f;
  if (gate_count && b == 0 && threadIdx.x == 0) *gate_count += 1u;
  const float2* p = partial + (size_t)b * n_tiles;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < n_tiles; i += 256) m = fmaxf(m, p[i].x);
  const float M = block_max(m, red);
  float s = 0.f;
  for (int i = threadIdx.x; i < n_tiles; i += 256) {
    const float2 v = p[i];
    if (v.x > -INFINITY) s += v.y * expf(v.x - M);
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float lse = M + logf(s);
    lse_out[b] = lse;
    loss_b[b] = lse - (true_logit ? true_logit[b] : S[(size_t)b * ldS + target[b]]);     // true_logit: the slab holds no logits
  }
}

// tl[b] = v_b . Ytab[target_b - row0]  (fp32), or 0 when the example's class is not one of this rank's Y rows: the true-class
// logit of the loss when the logits themselves are never written out (recompute_logits).  One warp per example.
__global__ void __launch_bounds__(256)
true_logit_kernel(const float* __restrict__ v, const float* __restrict__ Ytab, const int32_t* __restrict__ target, int row0, int Y,
                  int D, int B, float* __restrict__ tl, int* __restrict__ clear_flag = nullptr) {
  if (clear_flag && blockIdx.x == 0 && threadIdx.x == 0) *clear_flag = 0;      // the exp_slab range flag of the step that starts here
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  const int t = target[b] - row0;
  float acc = 0.f;
  if (t >= 0 && t < Y) {
    const float* y = Ytab + (size_t)t * D;
    const float* x = v + (size_t)b * D;
    for (int j = lane * 4; j < D; j += 128) {
      const float4 a = *reinterpret_cast<const float4*>(x + j), c = *reinterpret_cast<const float4*>(y + j);
      acc += a.x * c.x + a.y * c.y + a.z * c.z + a.w * c.w;
    }
    acc = warp_sum(acc);
  }
  if (lane == 0) tl[b] = acc;
}

// exp_slab schedule: the logits epilogue (umma::EpiExpSumT) left U = exp(s - c_b) in the slab and (max U, sum U) partials.
// Per example b, with Z = sum_j U[b, j]:  log-sum-exp = c_b + log Z,  loss_b = (c_b - true logit) + log Z,
// softmax - onehot = (U - Z [j == y_b]) / Z  -- so ONE element of the row is patched (U[b, y_b] -= Z) and the row's factor
// 1 / (B Z) (rscale) is handed to the two gradient GEMMs: it scales dv's rows in the split-K reduction and the code vectors
// that are dY's small operand (scale_rows_kernel).  A row whose largest U is outside [kExpSlabMin, kExpSlabMax] (or not a
// number), or whose scaled code vector rscale v_b has its largest element below kExpSlabMinOperand (common.cuh: smaller,
// and the tensor cores would read subnormal operands that keep only a few bits), raises *bad: the gated two-pass kernels
// that follow then redo the step's softmax the classic way.  One CTA per row.
__global__ void __launch_bounds__(256)
expsum_combine_kernel(const float2* __restrict__ partial, int n_tiles, float* __restrict__ U, float* __restrict__ U_lo, size_t ldS, int Y,
                      const int32_t* __restrict__ target, const float* __restrict__ offset, const float* __restrict__ true_logit,
                      const float* __restrict__ v, int D, float inv_batch, float* __restrict__ loss_b, float* __restrict__ lse_out,
                      float* __restrict__ rscale, int* __restrict__ bad) {
  __shared__ float red[32];
  const int b = blockIdx.x;
  const float2* p = partial + (size_t)b * n_tiles;
  float m = 0.f, s = 0.f, a = 0.f;
  for (int i = threadIdx.x; i < n_tiles; i += 256) {
    const float2 q = p[i];
    m = fmaxf(m, q.x);
    s += q.y;
  }
  for (int j = threadIdx.x; j < D; j += 256) a = fmaxf(a, fabsf(v[(size_t)b * D + j]));
  const float M = block_max(m, red);
  const float A = block_max(a, red);
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float r = inv_batch / s;
    if (!(M >= kExpSlabMin && M <= kExpSlabMax && s <= 3.0e38f)) *bad = 1;      // NaN fails every comparison
    if (A > 0.f && !(r * A >= kExpSlabMinOperand)) *bad = 1;                     // a zero code vector loses nothing
    const float lz = logf(s);
    lse_out[b] = offset[b] + lz;
    loss_b[b] = (offset[b] - true_logit[b]) + lz;
    rscale[b] = r;
    const int y = target[b];
    if (y >= 0 && y < Y) {
      const size_t at = (size_t)b * ldS + y;
      if (U_lo) {
        float hi, lo;
        split_tf32((U[at] + U_lo[at]) - s, hi, lo);
        U[at] = hi; U_lo[at] = lo;
      } else {
        U[at] -= s;
      }
    }
  }
}

// out[b, :] = x[b, :] * f[b]   (rows of length D; out may be x)
__global__ void __launch_bounds__(256)
scale_rows_kernel(const float* x, const float* __restrict__ f, float* out, int D, size_t n) {
  const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (i < n) out[i] = x[i] * f[i / D];
}

// exp_slab with a row-sharded target table (fully sharded schedule): this rank's slab holds U = exp(s - c_b) for its own classes,
// c_b = the example's true-class logit if that class lives here, else 0.  expsum_rows_kernel hands (c_b, sum U) to the
// cross-rank log-sum-exp in place of (row max, sum exp) -- the combine is the same formula -- and raises *bad when a row's
// largest U left the fp32 window.  One CTA per row.
__global__ void __launch_bounds__(256)
expsum_rows_kernel(const float2* __restrict__ partial, int n_tiles, const float* __restrict__ offset, float* __restrict__ row_max,
                   float* __restrict__ row_sum, int* __restrict__ bad) {
  __shared__ float red[32];
  const int b = blockIdx.x;
  const float2* p = partial + (size_t)b * n_tiles;
  float m = 0.f, s = 0.f;
  for (int i = threadIdx.x; i < n_tiles; i += 256) {
    const float2 q = p[i];
    m = fmaxf(m, q.x);
    s += q.y;
  }
  const float M = block_max(m, red);
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    if (!(M >= kExpSlabMin && M <= kExpSlabMax && s <= 3.0e38f)) *bad = 1;
    row_max[b] = offset[b];
    row_sum[b] = s;
  }
}
// ... and once the global log-sum-exp is known: softmax - onehot = f_b (U - [j == y_b] / f_b) with f_b = exp(c_b - lse_b); the one
// element is patched here and f_b / B becomes the row's factor for the gradient GEMMs.  A factor outside fp32's comfortable
// range raises *bad as well (the gated two-pass kernels behind this one then rebuild the slab).  One thread per row.
__global__ void __launch_bounds__(256)
expsum_finish_kernel(float* __restrict__ U, float* __restrict__ U_lo, size_t ldS, int Y, const int32_t* __restrict__ target, int row0,
                     const float* __restrict__ offset, const float* __restrict__ lse, float inv_batch, int Bt,
                     float* __restrict__ rscale, int* __restrict__ bad) {
  const int b = blockIdx.x * 256 + threadIdx.x;
  if (b >= Bt || *bad) return;
  const float d = offset[b] - lse[b];
  if (!(d > -80.f && d < 80.f)) { *bad = 1; return; }
  rscale[b] = inv_batch * expf(d);
  const int y = target[b] - row0;
  if (y >= 0 && y < Y) {
    const size_t at = (size_t)b * ldS + y;
    const float back = expf(-d);
    if (U_lo) {
      float hi, lo;
      split_tf32((U[at] + U_lo[at]) - back, hi, lo);
      U[at] = hi; U_lo[at] = lo;
    } else {
      U[at] -= back;
    }
  }
}

// S <- (softmax(S) - onehot(target)) * inv_batch in place, padding columns zeroed.  grid (chunks, B).
template <bool SPLIT>
__global__ void __launch_bounds__(256)
softmax_grad_kernel(float* __restrict__ S, size_t ldS, int Y, const float* __restrict__ lse, const int32_t* __restrict__ target,
                    float inv_batch, int row0, float* __restrict__ S_lo, const int* __restrict__ gate = nullptr,
                    float* __restrict__ rscale_one = nullptr, unsigned* __restrict__ gate_count = nullptr) {
  // SPLIT (3xTF32): the gradient is written as its tf32 split (high parts over S, residuals into S_lo)
  if (gate && *gate == 0) return;        // fallback pass of the exp_slab schedule: not needed this step
  if (rscale_one && blockIdx.x == 0 && threadIdx.x == 0) rscale_one[blockIdx.y] = 1.f;     // the slab will hold the finished gradient
  if (gate_count && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *gate_count += 1u;
  const int b = blockIdx.y;
  float* row = S + (size_t)b * ldS;
  const float l = lse[b];
  const int y = target[b] - row0;                    // outside [0, Y): the target row lives on another rank
  const int n4 = (int)(ldS >> 2);
  for (int q = blockIdx.x * 256 + threadIdx.x; q < n4; q += gridDim.x * 256) {
    const int j = 4 * q;
    float4 x = *reinterpret_cast<const float4*>(row + j);
    x.x = (j + 0 < Y) ? expf(x.x - l) * inv_batch : 0.f;
    x.y = (j + 1 < Y) ? expf(x.y - l) * inv_batch : 0.f;
    x.z = (j + 2 < Y) ? expf(x.z - l) * inv_batch : 0.f;
    x.w = (j + 3 < Y) ? expf(x.w - l) * inv_batch : 0.f;
    if (y >= j && y < j + 4) {
      if (y == j) x.x -= inv_batch; else if (y == j + 1) x.y -= inv_batch;
      else if (y == j + 2) x.z -= inv_batch; else x.w -= inv_batch;
    }
    if (SPLIT) {
      float4 hi, lo;
      split_tf32(x, hi, lo);
      *reinterpret_cast<float4*>(row + j) = hi;
      *reinterpret_cast<float4*>(S_lo + (size_t)b * ldS + j) = lo;
    } else {
      *reinterpret_cast<float4*>(row + j) = x;
    }
  }
}

// x -> (hi, lo) tf32 split of a whole buffer (3xTF32: TRANSFORM, the code vectors, the target table).
__global__ void __launch_bounds__(256)
split_tf32_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, size_t n4) {
  const size_t step = (size_t)gridDim.x * 256;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n4; i += step) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    float4 h, l;
    split_tf32(v, h, l);
    reinterpret_cast<float4*>(hi)[i] = h;
    reinterpret_cast<float4*>(lo)[i] = l;
  }
}

// xT[c, r] = x[r, c]: x is [rows, cols] row-major (pitch cols), xT is [cols, ldT].  Makes the K-major copy of a GEMM operand
// that is stored MN-major (TRANSFORM, the code vectors, the target table), so the GEMM reads it by TMA without transposing it in
// shared memory once per work item.  SPLIT (3xTF32): xT / xT_lo receive the transposed tf32 split, and hi / lo, when given, the
// untransposed one (x's layout, as split_tf32_kernel writes it).  Columns [rows, ldT) of xT are not written.  32 x 32 tiles,
// grid (ceil(rows / 32), ceil(cols / 32)).
template <bool SPLIT>
__global__ void __launch_bounds__(256)
transpose_kernel(const float* __restrict__ x, int rows, int cols, float* __restrict__ xT, float* __restrict__ xT_lo, size_t ldT,
                 float* __restrict__ hi, float* __restrict__ lo) {
  __shared__ float th[32][33];
  __shared__ float tl[SPLIT ? 32 : 1][33];
  const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int i = ty; i < 32; i += 8) {
    const int r = r0 + i, c = c0 + tx;
    if (r >= rows || c >= cols) continue;
    const size_t at = (size_t)r * cols + c;
    const float v = x[at];
    if constexpr (SPLIT) {
      float h, l;
      split_tf32(v, h, l);
      if (hi) { hi[at] = h; lo[at] = l; }
      th[i][tx] = h;
      tl[i][tx] = l;
    } else {
      th[i][tx] = v;
    }
  }
  __syncthreads();
#pragma unroll
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i, r = r0 + tx;
    if (r >= rows || c >= cols) continue;
    const size_t at = (size_t)c * ldT + r;
    xT[at] = th[tx][i];
    if constexpr (SPLIT) xT_lo[at] = tl[tx][i];
  }
}

// ---------------------------------------------------------------------------------------------
// Sampled softmax (BASELINE config 3; NOT in the reference, definition in DESIGN.md section 5 after
// tf.nn.sampled_softmax_loss): logits over {target_b} U sampled[0..S) minus log expected counts,
// accidental hits masked, cross entropy with the true class in column 0.  One CTA per example:
// logits, softmax, dl = (p - onehot)/B, loss_b and dv_b = sum_j dl_j * Ytab[row_j].
// ---------------------------------------------------------------------------------------------
constexpr int kSampledThreads = 128;
constexpr int kMaxSampled = 1024;

__global__ void __launch_bounds__(kSampledThreads)
sampled_softmax_fwd_kernel(const float* __restrict__ v, const float* __restrict__ Ytab, const int32_t* __restrict__ target,
                           const int32_t* __restrict__ sampled, int S, const float* __restrict__ logq_true,
                           const float* __restrict__ logq_samp, int D, float inv_batch, float* __restrict__ loss_b,
                           float* __restrict__ dl, float* __restrict__ dv) {
  extern __shared__ float sm[];
  float* vs = sm;                 // [D]
  float* lg = vs + D;             // [1 + S]
  __shared__ float red[32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int y = target[b];
  for (int i = tid; i < D; i += kSampledThreads) vs[i] = v[(size_t)b * D + i];
  __syncthreads();
  for (int j = warp; j <= S; j += kSampledThreads / 32) {
    const int row = (j == 0) ? y : sampled[j - 1];
    const float* r = Ytab + (size_t)row * D;
    float part = 0.f;
    for (int i = lane * 4; i < D; i += 128) {
      const float4 a = *reinterpret_cast<const float4*>(r + i);
      part += a.x * vs[i] + a.y * vs[i + 1] + a.z * vs[i + 2] + a.w * vs[i + 3];
    }
    part = warp_sum(part);
    if (lane == 0) {
      float l = part - ((j == 0) ? logq_true[b] : logq_samp[j - 1]);
      if (j > 0 && row == y) l = -1e9f;                     // accidental hit
      lg[j] = l;
    }
  }
  __syncthreads();
  float m = -INFINITY;
  for (int j = tid; j <= S; j += kSampledThreads) m = fmaxf(m, lg[j]);
  m = block_max(m, red);
  float s = 0.f;
  for (int j = tid; j <= S; j += kSampledThreads) s += expf(lg[j] - m);
  s = block_sum(s, red);
  const float lse = m + logf(s);
  if (tid == 0) loss_b[b] = lse - lg[0];
  __syncthreads();
  for (int j = tid; j <= S; j += kSampledThreads) {
    float g = expf(lg[j] - lse);
    if (j == 0) g -= 1.f;
    g *= inv_batch;
    if (j > 0 && sampled[j - 1] == y) g = 0.f;
    lg[j] = g;
    dl[(size_t)b * (S + 1) + j] = g;
  }
  __syncthreads();
  for (int i = tid; i < D; i += kSampledThreads) {
    float acc = lg[0] * Ytab[(size_t)y * D + i];
    for (int j = 1; j <= S; ++j) acc += lg[j] * Ytab[(size_t)sampled[j - 1] * D + i];
    dv[(size_t)b * D + i] = acc;
  }
}

// target-table gradient of the sampled softmax, added into gradient rows that are zero on entry:
// grid.x in [0, B): true rows  g[y_b] += dl[b,0] v_b ;
// grid.x in [B, B + S * chunks): g[sampled_s] += sum_{b in chunk} dl[b,1+s] v_b  (chunks of kSampledChunk examples, so the
// S sums spread over S * chunks blocks instead of S).
constexpr int kSampledChunk = 64;
__global__ void __launch_bounds__(kSampledThreads)
sampled_softmax_bwd_kernel(const float* __restrict__ v, const float* __restrict__ dl, const int32_t* __restrict__ target,
                           const int32_t* __restrict__ sampled, int B, int S, int D, float* __restrict__ g_tgt) {
  const int blk = blockIdx.x;
  if (blk < B) {
    const float g = dl[(size_t)blk * (S + 1)];
    float* dst = g_tgt + (size_t)target[blk] * D;
    for (int i = threadIdx.x; i < D; i += kSampledThreads) atomicAdd(dst + i, g * v[(size_t)blk * D + i]);
  } else {
    const int chunks = (B + kSampledChunk - 1) / kSampledChunk;
    const int s = (blk - B) / chunks, c = (blk - B) % chunks;
    const int b0 = c * kSampledChunk, b1 = min(B, b0 + kSampledChunk);
    float* dst = g_tgt + (size_t)sampled[s] * D;
    for (int i = threadIdx.x; i < D; i += kSampledThreads) {
      float acc = 0.f;
      for (int b = b0; b < b1; ++b) acc += dl[(size_t)b * (S + 1) + 1 + s] * v[(size_t)b * D + i];
      atomicAdd(dst + i, acc);
    }
  }
}

// Fully sharded schedule: this rank holds a row slice of the target table, so a row of S covers only
// its local classes.  row_maxsum_kernel: (max, sum exp) over the local columns -- from the logits
// epilogue's partial slots when present, else by scanning the row -- and the local true logit
// (S[b, t] if the example's target row lives here, else 0).  lse_combine_kernel folds the ranks'
// partials into the global log-sum-exp and the per-example loss.
__global__ void __launch_bounds__(256)
row_maxsum_kernel(const float2* __restrict__ partial, int slots, const float* __restrict__ S, size_t ldS, int Y,
                  const int32_t* __restrict__ target, int row0, float* __restrict__ row_max, float* __restrict__ row_sum,
                  float* __restrict__ true_logit, int have_true_logit = 0, const int* __restrict__ gate = nullptr) {
  // have_true_logit: true_logit[] was already filled by true_logit_kernel (the slab holds no logits)
  // gate: fallback launch of the exp_slab schedule, a no-op while *gate == 0
  if (gate && *gate == 0) return;
  __shared__ float red[32];
  const int b = blockIdx.x;
  const float* row = S + (size_t)b * ldS;
  float m = -INFINITY, s = 0.f;
  if (partial) {
    const float2* p = partial + (size_t)b * slots;
    for (int i = threadIdx.x; i < slots; i += 256) m = fmaxf(m, p[i].x);
    m = block_max(m, red);
    for (int i = threadIdx.x; i < slots; i += 256) {
      const float2 v = p[i];
      if (v.x > -INFINITY) s += v.y * expf(v.x - m);
    }
  } else {
    for (int j = threadIdx.x; j < Y; j += 256) m = fmaxf(m, row[j]);
    m = block_max(m, red);
    for (int j = threadIdx.x; j < Y; j += 256) s += expf(row[j] - m);
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    row_max[b] = m;
    row_sum[b] = s;
    if (target && !have_true_logit) {                // target == nullptr: the statistics only (c2v_topk_partial)
      const int t = target[b] - row0;                // local row of the example's target, if it lives here
      true_logit[b] = (t >= 0 && t < Y) ? row[t] : 0.f;
    }
  }
}

__global__ void __launch_bounds__(256)
lse_combine_kernel(const float* __restrict__ maxes, const float* __restrict__ sums, int world, int Bt,
                   const float* __restrict__ true_logit, float* __restrict__ lse_out, float* __restrict__ loss_b) {
  const int b = blockIdx.x * 256 + threadIdx.x;
  if (b >= Bt) return;
  float m = -INFINITY;
  for (int r = 0; r < world; ++r) m = fmaxf(m, maxes[(size_t)r * Bt + b]);
  float s = 0.f;
  for (int r = 0; r < world; ++r) {
    const float mr = maxes[(size_t)r * Bt + b];
    if (mr > -INFINITY) s += sums[(size_t)r * Bt + b] * expf(mr - m);
  }
  const float lse = m + logf(s);
  lse_out[b] = lse;
  loss_b[b] = lse - true_logit[b];
}

// loss = (sum_b loss_b) * inv_batch, fixed summation order.
__global__ void __launch_bounds__(256) loss_reduce_kernel(const float* __restrict__ loss_b, int B, float inv_batch,
                                                          float* __restrict__ out) {
  __shared__ float red[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < B; i += 256) s += loss_b[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) out[0] = s * inv_batch;
}

// out[j] = sum_{r<R} in[r*stride + j] for j < n   (split-K partials, per-example da partials).
// block (32, 32): thread (x, y) sums rows y, y+32, ...; fixed-order tree over y.
__global__ void __launch_bounds__(1024) colsum_kernel(const float* __restrict__ in, size_t stride, int R, int n,
                                                      float* __restrict__ out) {
  __shared__ float t[32][33];
  const int x = threadIdx.x, y = threadIdx.y;
  const int j = blockIdx.x * 32 + x;
  float s = 0.f;
  if (j < n)
    for (int r = y; r < R; r += 32) s += in[(size_t)r * stride + j];
  t[y][x] = s;
  __syncthreads();
  for (int o = 16; o > 0; o >>= 1) {
    if (y < o) t[y][x] += t[y + o][x];
    __syncthreads();
  }
  if (y == 0 && j < n) out[j] = t[0][x];
}

// out[i] = sum_{r<R} in[r*stride + i] for the few, long slices a split-K GEMM leaves behind
// (R <= ~64, n up to millions): one float4 column per thread, slices added in fixed order.
__global__ void __launch_bounds__(256)
slice_sum_kernel(const float* __restrict__ in, size_t stride, int R, size_t n4, float* __restrict__ out,
                 const float* __restrict__ row_scale = nullptr, int row_len4 = 1) {
  // row_scale: the result is a [rows, 4 * row_len4] matrix whose row i is multiplied by row_scale[i] on the way out
  const size_t step = (size_t)gridDim.x * 256;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n4; i += step) {
    float4 acc = reinterpret_cast<const float4*>(in)[i];
    for (int r = 1; r < R; ++r) {
      const float4 x = *reinterpret_cast<const float4*>(in + (size_t)r * stride + 4 * i);
      acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
    }
    if (row_scale) {
      const float f = row_scale[i / (size_t)row_len4];
      acc.x *= f; acc.y *= f; acc.z *= f; acc.w *= f;
    }
    reinterpret_cast<float4*>(out)[i] = acc;
  }
}

// ---------------------------------------------------------------------------------------------
// tf.nn.top_k over a row of scores: sorted descending, ties -> lower index   [TF-lib]
// (tensorflow_model.py:299-304); normalize: softmax over the k values (:305-306).
// ---------------------------------------------------------------------------------------------
constexpr int kTopkThreads = 256;

struct ValIdx { float v; int i; };
__device__ __forceinline__ bool better(float va, int ia, float vb, int ib) {   // a strictly before b
  return va > vb || (va == vb && ia < ib);
}
__device__ __forceinline__ ValIdx block_argbest(float v, int i, ValIdx* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (better(ov, oi, v, i)) { v = ov; i = oi; }
  }
  __syncthreads();
  if (lane == 0) { red[warp].v = v; red[warp].i = i; }
  __syncthreads();
  if (warp == 0) {
    v = (lane < kTopkThreads / 32) ? red[lane].v : -INFINITY;
    i = (lane < kTopkThreads / 32) ? red[lane].i : INT_MAX;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, v, o);
      const int oi = __shfl_xor_sync(0xffffffffu, i, o);
      if (better(ov, oi, v, i)) { v = ov; i = oi; }
    }
    if (lane == 0) { red[0].v = v; red[0].i = i; }
  }
  __syncthreads();
  ValIdx r = red[0];
  __syncthreads();
  return r;
}

__device__ __forceinline__ void topk_finish(float* vals, int k, int normalize, float* val_out) {
  // thread 0 only.  normalize: 0 raw logits; 1 softmax over the k values (tensorflow_model.py:305-306);
  // 2 raw here, topk_full_softmax_kernel turns them into full-vocabulary probabilities afterwards.
  if (normalize == 1) {
    float mx = vals[0], s = 0.f;
    for (int q = 0; q < k; ++q) s += expf(vals[q] - mx);
    for (int q = 0; q < k; ++q) val_out[q] = expf(vals[q] - mx) / s;
  } else {
    for (int q = 0; q < k; ++q) val_out[q] = vals[q];
  }
}

// Column j of a row-sharded slab whose first column is global class row_offset (c2v_topk_partial); the padding id INT_MAX
// stays INT_MAX
__device__ __forceinline__ int topk_global_id(int j, int row_offset) { return j == INT_MAX ? INT_MAX : j + row_offset; }

// Fast path, k <= K: per-thread sorted register list, then k rounds of block arg-best over the heads.
template <int K>
__global__ void __launch_bounds__(kTopkThreads)
topk_kernel(const float* __restrict__ S, size_t ldS, int Y, int k, int normalize, int32_t* __restrict__ idx_out,
            float* __restrict__ val_out, int row_offset = 0) {
  __shared__ ValIdx red[32];
  __shared__ float cv[kTopkThreads * K];
  __shared__ int ci[kTopkThreads * K];
  __shared__ float outv[K];
  const float* row = S + (size_t)blockIdx.x * ldS;
  const int tid = threadIdx.x;
  float tv[K];
  int ti[K];
#pragma unroll
  for (int q = 0; q < K; ++q) { tv[q] = -INFINITY; ti[q] = INT_MAX; }
  auto consider = [&](float x, int j) {
    if (x > tv[K - 1]) {
      tv[K - 1] = x; ti[K - 1] = j;
#pragma unroll
      for (int q = K - 1; q > 0; --q) {
        if (tv[q] > tv[q - 1]) {
          const float fv = tv[q]; tv[q] = tv[q - 1]; tv[q - 1] = fv;
          const int fi = ti[q]; ti[q] = ti[q - 1]; ti[q - 1] = fi;
        }
      }
    }
  };
  const int Y4 = Y >> 2;
  for (int q = tid; q < Y4; q += kTopkThreads) {
    const float4 x = *reinterpret_cast<const float4*>(row + 4 * q);
    consider(x.x, 4 * q); consider(x.y, 4 * q + 1); consider(x.z, 4 * q + 2); consider(x.w, 4 * q + 3);
  }
  for (int j = 4 * Y4 + tid; j < Y; j += kTopkThreads) consider(row[j], j);
#pragma unroll
  for (int q = 0; q < K; ++q) { cv[tid * K + q] = tv[q]; ci[tid * K + q] = ti[q]; }
  int head = 0;
  for (int r = 0; r < k; ++r) {
    const float hv = (head < K) ? cv[tid * K + head] : -INFINITY;
    const int hi = (head < K) ? ci[tid * K + head] : INT_MAX;
    const ValIdx w = block_argbest(hv, hi, red);
    if (w.i == hi && hi != INT_MAX) ++head;
    if (tid == 0) { idx_out[(size_t)blockIdx.x * k + r] = topk_global_id(w.i, row_offset); outv[r] = w.v; }
  }
  if (tid == 0) topk_finish(outv, k, normalize, val_out + (size_t)blockIdx.x * k);
}

// General path (any k <= 64): k rounds, each a block arg-best over the entries ordered after
// the previous pick.
__global__ void __launch_bounds__(kTopkThreads)
topk_iter_kernel(const float* __restrict__ S, size_t ldS, int Y, int k, int normalize, int32_t* __restrict__ idx_out,
                 float* __restrict__ val_out, int row_offset = 0) {
  __shared__ ValIdx red[32];
  __shared__ float outv[64];
  const float* row = S + (size_t)blockIdx.x * ldS;
  const int tid = threadIdx.x;
  float pv = INFINITY;
  int pi = -1;
  for (int r = 0; r < k; ++r) {
    float bv = -INFINITY;
    int bi = INT_MAX;
    for (int j = tid; j < Y; j += kTopkThreads) {
      const float x = row[j];
      const bool after = (x < pv) || (x == pv && j > pi);
      if (after && better(x, j, bv, bi)) { bv = x; bi = j; }
    }
    const ValIdx w = block_argbest(bv, bi, red);
    pv = w.v; pi = w.i;
    if (tid == 0) { idx_out[(size_t)blockIdx.x * k + r] = topk_global_id(w.i, row_offset); outv[r] = w.v; }
  }
  if (tid == 0) topk_finish(outv, k, normalize, val_out + (size_t)blockIdx.x * k);
}

// normalize == 2: the Keras backend's scores (keras_model.py:69-70, keras_topk_word_predictions_layer.py:30-35):
// top-k of softmax(logits) over the WHOLE target vocabulary.  softmax is monotone, so the indices are
// those of the logits; the k values become exp(l - max) / sum_j exp(l_j - max).
__global__ void __launch_bounds__(256)
topk_full_softmax_kernel(const float* __restrict__ S, size_t ldS, int Y, int k, float* __restrict__ val) {
  __shared__ float red[32];
  const float* row = S + (size_t)blockIdx.x * ldS;
  float m = -INFINITY, s = 0.f;
  for (int j = threadIdx.x; j < Y; j += 256) m = fmaxf(m, row[j]);
  m = block_max(m, red);
  for (int j = threadIdx.x; j < Y; j += 256) s += expf(row[j] - m);
  s = block_sum(s, red);
  if (threadIdx.x < k) {
    float* v = val + (size_t)blockIdx.x * k + threadIdx.x;
    *v = expf(*v - m) / s;
  }
}

// ---------------------------------------------------------------------------------------------
// Merge of sorted candidate lists (c2v_topk_partial over a rank's partial slots, c2v_topk_merge across ranks).  Output
// row b takes input row row0 + b: L lists of k (value, global id) pairs, list l at (row0 + b) * row_stride + l * list_stride,
// each sorted by `better` with its padding (-inf, INT_MAX) last, and keeps the best k of their union in the same order.
// Every element of a row's top k is in the top k of the list that holds it, so the result is the top k of the whole row
// under tf.nn.top_k's order.  normalize 0 / 1: topk_finish; 2: exp(v - M) / S, (M, S) the combine of the ranks'
// (max, sum exp) pairs maxes / sums [world, Bt] as in lse_combine_kernel.
// ---------------------------------------------------------------------------------------------
struct TopkMergeArgs {
  const int32_t* idx;
  const float* val;
  int L;
  size_t row_stride, list_stride;
  int k, normalize;
  const float* maxes;       // normalize 2: [world, Bt]
  const float* sums;
  int world, Bt, row0;
  int32_t* idx_out;         // [rows, k]
  float* val_out;
};

__device__ __forceinline__ void topk_merge_finish(const TopkMergeArgs& a, float* vals) {
  // thread 0 only
  const int row = a.row0 + blockIdx.x;
  float* out = a.val_out + (size_t)blockIdx.x * a.k;
  if (a.normalize != 2) { topk_finish(vals, a.k, a.normalize, out); return; }
  float m = -INFINITY;
  for (int r = 0; r < a.world; ++r) m = fmaxf(m, a.maxes[(size_t)r * a.Bt + row]);
  float s = 0.f;
  for (int r = 0; r < a.world; ++r) {
    const float mr = a.maxes[(size_t)r * a.Bt + row];
    if (mr > -INFINITY) s += a.sums[(size_t)r * a.Bt + row] * expf(mr - m);
  }
  for (int q = 0; q < a.k; ++q) out[q] = expf(vals[q] - m) / s;
}

// k <= K: each thread keeps a sorted register list of the best K entries of its lists (a list is read only while its
// entries still enter), then k rounds of block arg-best over the threads' heads, as topk_kernel.
template <int K>
__global__ void __launch_bounds__(kTopkThreads) topk_merge_kernel(TopkMergeArgs a) {
  __shared__ ValIdx red[32];
  __shared__ float cv[kTopkThreads * K];
  __shared__ int ci[kTopkThreads * K];
  __shared__ float outv[K];
  const int tid = threadIdx.x;
  const size_t row = (size_t)(a.row0 + blockIdx.x) * a.row_stride;
  float tv[K];
  int ti[K];
#pragma unroll
  for (int q = 0; q < K; ++q) { tv[q] = -INFINITY; ti[q] = INT_MAX; }
  for (int l = tid; l < a.L; l += kTopkThreads) {
    const float* lv = a.val + row + (size_t)l * a.list_stride;
    const int32_t* li = a.idx + row + (size_t)l * a.list_stride;
    for (int q = 0; q < a.k; ++q) {
      const float x = lv[q];
      const int j = li[q];
      if (!better(x, j, tv[K - 1], ti[K - 1])) break;      // the list is sorted: none of its later entries enters either
      tv[K - 1] = x; ti[K - 1] = j;
#pragma unroll
      for (int p = K - 1; p > 0; --p) {
        if (better(tv[p], ti[p], tv[p - 1], ti[p - 1])) {
          const float fv = tv[p]; tv[p] = tv[p - 1]; tv[p - 1] = fv;
          const int fi = ti[p]; ti[p] = ti[p - 1]; ti[p - 1] = fi;
        }
      }
    }
  }
#pragma unroll
  for (int q = 0; q < K; ++q) { cv[tid * K + q] = tv[q]; ci[tid * K + q] = ti[q]; }
  int head = 0;
  for (int r = 0; r < a.k; ++r) {
    const float hv = (head < K) ? cv[tid * K + head] : -INFINITY;
    const int hi = (head < K) ? ci[tid * K + head] : INT_MAX;
    const ValIdx w = block_argbest(hv, hi, red);
    if (w.i == hi && hi != INT_MAX) ++head;
    if (tid == 0) { a.idx_out[(size_t)blockIdx.x * a.k + r] = w.i; outv[r] = w.v; }
  }
  if (tid == 0) topk_merge_finish(a, outv);
}

// Any k <= 64 (the slab route's k > 16, L = world): k rounds, each a block arg-best over the entries ordered after the
// previous pick, as topk_iter_kernel.
__global__ void __launch_bounds__(kTopkThreads) topk_merge_iter_kernel(TopkMergeArgs a) {
  __shared__ ValIdx red[32];
  __shared__ float outv[64];
  const int tid = threadIdx.x;
  const size_t row = (size_t)(a.row0 + blockIdx.x) * a.row_stride;
  const int n = a.L * a.k;
  float pv = INFINITY;
  int pi = -1;
  for (int r = 0; r < a.k; ++r) {
    float bv = -INFINITY;
    int bi = INT_MAX;
    for (int e = tid; e < n; e += kTopkThreads) {
      const size_t off = row + (size_t)(e / a.k) * a.list_stride + e % a.k;
      const float x = a.val[off];
      const int j = a.idx[off];
      if (better(pv, pi, x, j) && better(x, j, bv, bi)) { bv = x; bi = j; }
    }
    const ValIdx w = block_argbest(bv, bi, red);
    pv = w.v; pi = w.i;
    if (tid == 0) { a.idx_out[(size_t)blockIdx.x * a.k + r] = w.i; outv[r] = w.v; }
  }
  if (tid == 0) topk_merge_finish(a, outv);
}

// ---------------------------------------------------------------------------------------------
// tf.compat.v1.train.AdamOptimizer dense apply (tensorflow_model.py:232; SURVEY A.3).  Every
// element is visited (TF1's sparse apply decays m, v and moves theta on all rows).  The operations
// and their order are the float32 step of tests/adam_model.py, with lr_t computed on the host as
// oracle.adam_lr_t states it; tests/test_gpu_adam_model.py compares the bits.  zero_grad: clear g
// after use, so the next step's scatter-add starts from zero without a separate memset pass.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, size_t n4,
            float lr_t, float b1, float b2, float eps, int zero_grad) {
  const float omb1 = __fsub_rn(1.f, b1), omb2 = __fsub_rn(1.f, b2);
  auto upd = [&](float& pp, float gg, float& mm, float& vv) {
    mm = __fadd_rn(__fmul_rn(mm, b1), __fmul_rn(omb1, gg));
    vv = __fadd_rn(__fmul_rn(vv, b2), __fmul_rn(omb2, __fmul_rn(gg, gg)));
    pp = adam_move_dense(pp, lr_t, mm, vv, eps);
  };
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 P = reinterpret_cast<float4*>(p)[i];
    const float4 G = reinterpret_cast<const float4*>(g)[i];
    float4 Mm = reinterpret_cast<float4*>(m)[i];
    float4 V = reinterpret_cast<float4*>(v)[i];
    upd(P.x, G.x, Mm.x, V.x); upd(P.y, G.y, Mm.y, V.y); upd(P.z, G.z, Mm.z, V.z); upd(P.w, G.w, Mm.w, V.w);
    reinterpret_cast<float4*>(p)[i] = P;
    reinterpret_cast<float4*>(m)[i] = Mm;
    reinterpret_cast<float4*>(v)[i] = V;
    if (zero_grad) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// ---------------------------------------------------------------------------------------------
// tf32 path only: materialise the gathered, dropped-out context matrix once per step
//   X'[n, :] = dropout([ tok[src[n]] | path[pth[n]] | tok[tgt[n]] ])   (tensorflow_model.py:238-246)
// so the three projection GEMMs can be fed by TMA; and its inverse, the scatter-add of dX' rows
// into the embedding gradient tables.  One warp per context row, 128-bit accesses.
// ---------------------------------------------------------------------------------------------
template <bool SPLIT>
__global__ void __launch_bounds__(256)
gather_ctx_kernel(const __grid_constant__ ContextSource cs, const __grid_constant__ Dropout dp, float* __restrict__ Xg,
                  float* __restrict__ Xlo) {
  // SPLIT (3xTF32): X' is written as its tf32 split (high parts into Xg, residuals into Xlo)
  // Launched as one resident wave (gather_blocks()): a warp walks rows n, n + stride, ... and loads the three indices of
  // its NEXT row before it touches the current one, so a row costs one dependent memory round trip (the table rows),
  // not two (index, then rows).
  const int lane = threadIdx.x & 31;
  const int stride = gridDim.x * 8;
  int n = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (n >= cs.rows) return;
  const int K3 = 3 * cs.d;
  int i0 = __ldg(cs.src + n), i1 = __ldg(cs.pth + n), i2 = __ldg(cs.tgt + n);
  for (; n < cs.rows; n += stride) {
    const int nn = n + stride;
    int p0 = 0, p1 = 0, p2 = 0;
    if (nn < cs.rows) { p0 = __ldg(cs.src + nn); p1 = __ldg(cs.pth + nn); p2 = __ldg(cs.tgt + nn); }
    const float* r0 = table_row(cs.tok, i0, cs.d);
    const float* r1 = table_row(cs.path, i1, cs.d);
    const float* r2 = table_row(cs.tok, i2, cs.d);
    float* dst = Xg + (size_t)n * K3;
    // all loads of the row are issued before any is consumed: with peer (NVLink) shards each load is a
    // multi-microsecond round trip, so memory-level parallelism per warp is what sets the bandwidth
    constexpr int kU = 3;                          // covers 3d <= 384 (d = 128) in one batch
    for (int j0 = lane * 4; j0 < K3; j0 += 128 * kU) {
      float4 x[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int j = j0 + u * 128;
        if (j < K3) {
          const int seg = j / cs.d, off = j - seg * cs.d;
          const float* r = seg == 0 ? r0 : (seg == 1 ? r1 : r2);
          x[u] = __ldg(reinterpret_cast<const float4*>(r + off));
        }
      }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int j = j0 + u * 128;
        if (j < K3) {
          const float4 m = dropout_mult4(dp, n, j >> 2);
          x[u].x *= m.x; x[u].y *= m.y; x[u].z *= m.z; x[u].w *= m.w;
          if (SPLIT) {
            float4 hi, lo;
            split_tf32(x[u], hi, lo);
            *reinterpret_cast<float4*>(dst + j) = hi;
            *reinterpret_cast<float4*>(Xlo + (size_t)n * K3 + j) = lo;
          } else {
            *reinterpret_cast<float4*>(dst + j) = x[u];
          }
        }
      }
    }
    i0 = p0; i1 = p1; i2 = p2;
  }
}

__global__ void __launch_bounds__(256)
scatter_dx_kernel(const __grid_constant__ ContextSource cs, const __grid_constant__ Dropout dp, const float* __restrict__ mask,
                  const float* __restrict__ dXg, const __grid_constant__ ShardedTable g_tok,
                  const __grid_constant__ ShardedTable g_path, float grad_scale) {
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= cs.rows) return;
  if (mask[n] == 0.f) return;                 // masked contexts carry exact zeros
  const int K3 = 3 * cs.d;
  const float* src = dXg + (size_t)n * K3;
  for (int j = lane * 4; j < K3; j += 128) {
    float4 g = *reinterpret_cast<const float4*>(src + j);
    const float4 m = dropout_mult4(dp, n, j >> 2);
    g.x *= m.x * grad_scale; g.y *= m.y * grad_scale; g.z *= m.z * grad_scale; g.w *= m.w * grad_scale;
    const int seg = j / cs.d, off = j - seg * cs.d;
    float* dst;
    if (seg == 0) dst = table_row(g_tok, cs.src[n], cs.d) + off;
    else if (seg == 1) dst = table_row(g_path, cs.pth[n], cs.d) + off;
    else dst = table_row(g_tok, cs.tgt[n], cs.d) + off;
    atomicAdd(reinterpret_cast<float4*>(dst), g);
  }
}

// ---------------------------------------------------------------------------------------------
// Row-sharded tables (peer memory over NVLink): locality-sorted gather / scatter-add.
//
// With the tables of BASELINE configs[4] (3M x 256 and 2M x 256 floats: 5 GB of parameters and 5 GB of gradient
// shards mapped from the peers) random row accesses to peer memory are TLB-bound: every access touches a different
// 2 MB page of a mapping far larger than the GPU's TLB reach.
// The context entries (n, segment) of a batch are therefore bucketed by (owner rank, 2 MB page of the owner's shard)
// with a counting sort -- bucket_count / bucket_scan / bucket_fill -- and the gather and the scatter-add walk the
// entries in bucket order: each remote page is visited once, by neighbouring warps, instead of once per access.
// The order inside a bucket is whatever the atomics give; it only changes the order of accesses, not any result
// (the scatter-add's float atomics are order-free up to rounding, as before).
// ---------------------------------------------------------------------------------------------
constexpr int kMaxBuckets = 8192;

struct BucketPlan {
  int shift, mask;          // as ShardedTable: owner = idx & mask, local row = idx >> shift
  int page_shift;           // rows per 2 MB page = 1 << page_shift
  int pages_tok, pages_path;   // pages per shard
  int n_buckets;            // (mask + 1) * (pages_tok + pages_path)
};
__device__ __forceinline__ int bucket_of(const BucketPlan& bp, int seg, int idx) {
  const int owner = idx & bp.mask, page = (idx >> bp.shift) >> bp.page_shift;
  return (seg == 1) ? (bp.mask + 1) * bp.pages_tok + owner * bp.pages_path + page : owner * bp.pages_tok + page;
}
__device__ __forceinline__ int entry_index(const ContextSource& cs, int e) {      // e = 3 n + seg
  const int n = e / 3, seg = e - 3 * n;
  return seg == 0 ? cs.src[n] : (seg == 1 ? cs.pth[n] : cs.tgt[n]);
}

__global__ void __launch_bounds__(256)
bucket_count_kernel(const __grid_constant__ ContextSource cs, const __grid_constant__ BucketPlan bp, int32_t* __restrict__ counts) {
  extern __shared__ int32_t hist[];
  for (int i = threadIdx.x; i < bp.n_buckets; i += 256) hist[i] = 0;
  __syncthreads();
  const int total = 3 * cs.rows;
  for (int e = blockIdx.x * 256 + threadIdx.x; e < total; e += gridDim.x * 256) {
    const int n = e / 3, seg = e - 3 * n;
    atomicAdd(&hist[bucket_of(bp, seg, entry_index(cs, e))], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < bp.n_buckets; i += 256)
    if (hist[i]) atomicAdd(&counts[i], hist[i]);
}

// exclusive scan of counts[0, n) into cursor[0, n) and starts[0, n] (one block); counts are cleared for the next batch
__global__ void __launch_bounds__(1024)
bucket_scan_kernel(int32_t* __restrict__ counts, int32_t* __restrict__ cursor, int32_t* __restrict__ starts, int n) {
  __shared__ int32_t part[1024];
  const int per = (n + 1023) / 1024;
  const int lo = threadIdx.x * per, hi = min(n, lo + per);
  int s = 0;
  for (int i = lo; i < hi; ++i) s += counts[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const int v = (threadIdx.x >= o) ? part[threadIdx.x - o] : 0;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  int run = part[threadIdx.x] - s;
  for (int i = lo; i < hi; ++i) {
    const int c = counts[i];
    cursor[i] = run;
    starts[i] = run;
    run += c;
    counts[i] = 0;
  }
  if (threadIdx.x == 1023) starts[n] = part[1023];      // total number of entries
}

__global__ void __launch_bounds__(256)
bucket_fill_kernel(const __grid_constant__ ContextSource cs, const __grid_constant__ BucketPlan bp, int32_t* __restrict__ cursor,
                   int32_t* __restrict__ perm) {
  const int total = 3 * cs.rows;
  for (int e = blockIdx.x * 256 + threadIdx.x; e < total; e += gridDim.x * 256) {
    const int n = e / 3, seg = e - 3 * n;
    perm[atomicAdd(&cursor[bucket_of(bp, seg, entry_index(cs, e))], 1)] = e;
  }
}

// X'[n, seg*d : (seg+1)*d] = dropout(table row) for the entries in bucket order; one warp per entry.
template <bool SPLIT>
__global__ void __launch_bounds__(256)
gather_sorted_kernel(const __grid_constant__ ContextSource cs, const __grid_constant__ Dropout dp, const int32_t* __restrict__ perm,
                     float* __restrict__ Xg, float* __restrict__ Xlo) {
  const int w = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= 3 * cs.rows) return;
  const int e = perm[w];
  const int n = e / 3, seg = e - 3 * n;
  const int idx = seg == 0 ? cs.src[n] : (seg == 1 ? cs.pth[n] : cs.tgt[n]);
  const float* row = (seg == 1) ? table_row(cs.path, idx, cs.d) : table_row(cs.tok, idx, cs.d);
  const size_t o = (size_t)n * (3 * cs.d) + (size_t)seg * cs.d;
  constexpr int kU = 2;                          // d <= 256 in one batch of loads
  for (int j0 = lane * 4; j0 < cs.d; j0 += 128 * kU) {
    float4 x[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u)
      if (j0 + u * 128 < cs.d) x[u] = __ldg(reinterpret_cast<const float4*>(row + j0 + u * 128));
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int j = j0 + u * 128;
      if (j < cs.d) {
        const float4 m = dropout_mult4(dp, n, (seg * cs.d + j) >> 2);
        x[u].x *= m.x; x[u].y *= m.y; x[u].z *= m.z; x[u].w *= m.w;
        if (SPLIT) {
          float4 hi, lo;
          split_tf32(x[u], hi, lo);
          *reinterpret_cast<float4*>(Xg + o + j) = hi;
          *reinterpret_cast<float4*>(Xlo + o + j) = lo;
        } else {
          *reinterpret_cast<float4*>(Xg + o + j) = x[u];
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256)
scatter_sorted_kernel(const __grid_constant__ ContextSource cs, const __grid_constant__ Dropout dp, const float* __restrict__ mask,
                      const int32_t* __restrict__ perm, const float* __restrict__ dXg, const __grid_constant__ ShardedTable g_tok,
                      const __grid_constant__ ShardedTable g_path, float grad_scale) {
  const int w = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= 3 * cs.rows) return;
  const int e = perm[w];
  const int n = e / 3, seg = e - 3 * n;
  if (mask[n] == 0.f) return;                 // masked contexts carry exact zeros
  const int idx = seg == 0 ? cs.src[n] : (seg == 1 ? cs.pth[n] : cs.tgt[n]);
  float* row = (seg == 1) ? table_row(g_path, idx, cs.d) : table_row(g_tok, idx, cs.d);
  const float* src = dXg + (size_t)n * (3 * cs.d) + (size_t)seg * cs.d;
  for (int j = lane * 4; j < cs.d; j += 128) {
    float4 g = *reinterpret_cast<const float4*>(src + j);
    const float4 m = dropout_mult4(dp, n, (seg * cs.d + j) >> 2);
    g.x *= m.x * grad_scale; g.y *= m.y * grad_scale; g.z *= m.z * grad_scale; g.w *= m.w * grad_scale;
    atomicAdd(reinterpret_cast<float4*>(row + j), g);
  }
}

// ---- push-based gradient exchange (c2v_bind_scatter_inbox) -------------------------------------------------------
// Inbox of one rank: [counts: 2 ints per sender, padded to 256 B][row ids: world x cap ints][values: world x cap x d floats]
// with cap = 3 * max_batch * max_contexts (a sender can never have more entries).  Sender s owns slots [s*cap, (s+1)*cap):
// its token-table rows first (count[2s]), then its path-table rows (count[2s+1]).
struct InboxView {
  int32_t* cnt;
  int32_t* ids;
  float* val;
};
__host__ __device__ inline size_t inbox_ids_offset(int world) { return ((size_t)world * 2 * 4 + 255) / 256 * 256; }
__host__ __device__ inline size_t inbox_val_offset(int world, size_t cap) {
  return (inbox_ids_offset(world) + (size_t)world * cap * 4 + 255) / 256 * 256;
}
struct InboxSet {
  char* base[kMaxShards];    // every rank's inbox as mapped here
  size_t cap;
  int world, rank;
};
__device__ __forceinline__ InboxView inbox_of(const InboxSet& s, int owner) {
  InboxView v;
  v.cnt = reinterpret_cast<int32_t*>(s.base[owner]);
  v.ids = reinterpret_cast<int32_t*>(s.base[owner] + inbox_ids_offset(s.world));
  v.val = reinterpret_cast<float*>(s.base[owner] + inbox_val_offset(s.world, s.cap));
  return v;
}

// starts[b] = first sorted position of bucket b (bucket_scan_kernel); the buckets of owner o are contiguous per table.
__global__ void inbox_counts_kernel(const __grid_constant__ InboxSet inbox, const __grid_constant__ BucketPlan bp,
                                    const int32_t* __restrict__ starts) {
  const int o = threadIdx.x;
  if (o > bp.mask) return;
  const int W = bp.mask + 1, t0 = o * bp.pages_tok, p0 = W * bp.pages_tok + o * bp.pages_path;
  InboxView v = inbox_of(inbox, o);
  v.cnt[2 * inbox.rank] = starts[t0 + bp.pages_tok] - starts[t0];
  v.cnt[2 * inbox.rank + 1] = starts[p0 + bp.pages_path] - starts[p0];
}

// one warp per sorted entry: the (dropout-scaled) gradient row goes into the owner's inbox, densely
__global__ void __launch_bounds__(256)
scatter_inbox_kernel(const __grid_constant__ ContextSource cs, const __grid_constant__ Dropout dp, const float* __restrict__ mask,
                     const int32_t* __restrict__ perm, const int32_t* __restrict__ starts, const __grid_constant__ BucketPlan bp,
                     const float* __restrict__ dXg, const __grid_constant__ InboxSet inbox, float grad_scale) {
  const int w = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= 3 * cs.rows) return;
  const int e = perm[w];
  const int n = e / 3, seg = e - 3 * n;
  const int idx = seg == 0 ? cs.src[n] : (seg == 1 ? cs.pth[n] : cs.tgt[n]);
  const int o = idx & bp.mask, W = bp.mask + 1;
  const int t0 = o * bp.pages_tok, p0 = W * bp.pages_tok + o * bp.pages_path;
  const int k = (seg == 1) ? (starts[t0 + bp.pages_tok] - starts[t0]) + (w - starts[p0]) : (w - starts[t0]);
  InboxView v = inbox_of(inbox, o);
  const size_t slot = (size_t)inbox.rank * inbox.cap + k;
  const bool live = mask[n] != 0.f;           // masked contexts carry exact zeros: the owner skips the slot
  if (lane == 0) v.ids[slot] = live ? (idx >> bp.shift) : -1;
  if (!live) return;
  const float* src = dXg + (size_t)n * (3 * cs.d) + (size_t)seg * cs.d;
  float* dst = v.val + slot * cs.d;
  for (int j = lane * 4; j < cs.d; j += 128) {
    float4 g = *reinterpret_cast<const float4*>(src + j);
    const float4 m = dropout_mult4(dp, n, (seg * cs.d + j) >> 2);
    g.x *= m.x * grad_scale; g.y *= m.y * grad_scale; g.z *= m.z * grad_scale; g.w *= m.w * grad_scale;
    *reinterpret_cast<float4*>(dst + j) = g;
  }
}

// the owner folds its inbox into its own gradient shards (local atomics); persistent grid, one warp per slot
__global__ void __launch_bounds__(256)
inbox_apply_kernel(const __grid_constant__ InboxSet inbox, int d, float* __restrict__ g_tok, float* __restrict__ g_path) {
  const int lane = threadIdx.x & 31;
  const int warp_global = (blockIdx.x * 256 + threadIdx.x) >> 5, total_warps = (gridDim.x * 256) >> 5;
  InboxView v = inbox_of(inbox, inbox.rank);
  for (int s = 0; s < inbox.world; ++s) {
    const int n_tok = v.cnt[2 * s], n_all = n_tok + v.cnt[2 * s + 1];
    for (int k = warp_global; k < n_all; k += total_warps) {
      const size_t slot = (size_t)s * inbox.cap + k;
      const int row = v.ids[slot];
      if (row < 0) continue;
      float* dst = (k < n_tok ? g_tok : g_path) + (size_t)row * d;
      const float* src = v.val + slot * d;
      for (int j = lane * 4; j < d; j += 128) atomicAdd(reinterpret_cast<float4*>(dst + j), *reinterpret_cast<const float4*>(src + j));
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Lazy-but-exact dense Adam for the two embedding tables (single GPU).
//
// TF1's Adam is dense: every row decays m, v and moves theta on every step, gradient or not
// (SURVEY A.3).  The update of a row depends only on (theta, m, v, g, step), and nothing reads a row
// between two batches that reference it, so the whole update can be DEFERRED without changing a
// single bit: each row remembers the last step it is current for (`last`); its gradient row keeps
// the scatter-add of the step that last touched it (zeros otherwise); and the pending steps are
// replayed -- same fp32 operations, same order: one step with that gradient, then zero-gradient
// steps -- the next time the row is about to be read (forward gather of a batch that references it).
// Per step only the rows of the current batch are touched (~25 % of the tables at B = 1024 x 200
// uniform, far fewer on Zipfian data), ONCE, instead of streaming 9 GB of theta / m / v.
//   mark_rows_kernel         : stamp[row] = epoch for every row the batch references
//   adam_rows_kernel<CATCHUP>: stamped rows -> replay steps last+1 .. t_done, clear the gradient row
//   adam_rows_kernel<FLUSH>  : all rows     -> the same (before export / checkpoint / mode switch)
// lr_tab[s & kLrRingMask] holds lr_s = lr*sqrt(1-b2^s)/(1-b1^s) as computed on the host for the dense kernel.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
mark_rows_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ pth, const int32_t* __restrict__ tgt, int n,
                 int32_t* __restrict__ stamp_tok, int32_t* __restrict__ stamp_path, int32_t epoch) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  stamp_tok[src[i]] = epoch;
  stamp_path[pth[i]] = epoch;
  stamp_tok[tgt[i]] = epoch;
}

// stamp[idx[i]] = epoch: the rows a sampled-softmax step reads from the target table
__global__ void __launch_bounds__(256)
mark_list_kernel(const int32_t* __restrict__ idx, int n, int32_t* __restrict__ stamp, int32_t epoch) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < n) stamp[idx[i]] = epoch;
}

__global__ void fill_i32_kernel(int32_t* __restrict__ p, size_t n, int32_t v) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void set_float_kernel(float* p, float v) { *p = v; }

enum { ADAM_ROWS_CATCHUP = 0, ADAM_ROWS_FLUSH = 2 };

// lr_tab is a ring over the step count: entry s & kLrRingMask holds lr_s.  No row is ever more than the
// ring's length behind: the engine sweeps a 1/R slice of every table per step (option "adam_sweep_period")
// and otherwise flushes all rows before the ring wraps.
constexpr int kLrRing = 1 << 16;
constexpr int kLrRingMask = kLrRing - 1;

// One row's pending steps last+1 .. t_done, by the whole warp (lane -> 4 consecutive elements of every
// 128-column slice): the first with whatever the gradient row holds -- the scatter-add of the step that last
// touched the row, or zeros -- and the rest with a zero gradient, in the dense kernel's operations and order;
// the gradient row is cleared on the way.
//
// "theta rests" exit (rest_ok): in a zero-gradient step m shrinks by b1 (~0.9) while sqrt(v) + eps shrinks by
// at most sqrt(b2) (~0.9995) and lr_s grows by less than 1.3 % per step (s >= 2), so the update
// delta_s = lr_s m_s / (sqrt(v_s) + eps) shrinks monotonically in magnitude and keeps its sign.  Rounding is
// monotone, so once fl(theta - delta_s) == theta for EVERY element of the row it stays so for all later steps:
// theta is left alone and only m <- fl(m b1), v <- fl(v b2) continue, without the division and square root.
// Bit-identical to the dense kernel: tests/test_lazy_adam_model.py checks the scheme on the CPU and
// tests/test_gpu_adam_model.py every element of the replayed tables against the float32 step on the GPU; the engine
// enables it only for 0 < b1 <= 0.95, 0.99 <= b2 < 1, eps > 0.  pos_eps: eps > 0 (adam_move's zero-numerator exit).
__device__ __forceinline__ void replay_row(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                           size_t row_off, int d, int32_t from, int32_t t_done, const float* __restrict__ lr_tab,
                                           float b1, float b2, float eps, float omb1, float omb2, int lane, bool rest_ok,
                                           bool pos_eps) {
  for (int j0 = 0; j0 < d; j0 += 128) {          // every lane walks every slice: the vote below needs all 32
    const int j = j0 + lane * 4;
    const bool act = j < d;
    const size_t o = row_off + (act ? j : 0);
    float4 P = make_float4(0.f, 0.f, 0.f, 0.f), M = P, V = P, G = P;
    if (act) {
      P = *reinterpret_cast<float4*>(p + o); M = *reinterpret_cast<float4*>(m + o); V = *reinterpret_cast<float4*>(v + o);
      G = *reinterpret_cast<const float4*>(g + o);
    }
    float* pp = reinterpret_cast<float*>(&P);
    float* mm = reinterpret_cast<float*>(&M);
    float* vv = reinterpret_cast<float*>(&V);
    const float* gg = reinterpret_cast<const float*>(&G);
    {  // step from+1: the deferred gradient step (the dense kernel's exact operations)
      const float lr_s = lr_tab[(from + 1) & kLrRingMask];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        mm[q] = __fadd_rn(__fmul_rn(mm[q], b1), __fmul_rn(omb1, gg[q]));
        vv[q] = __fadd_rn(__fmul_rn(vv[q], b2), __fmul_rn(omb2, __fmul_rn(gg[q], gg[q])));
        pp[q] = adam_move(pp[q], lr_s, mm[q], vv[q], eps, pos_eps);
      }
    }
    // the zero-gradient steps after it: m*b1 + (1-b1)*0, v*b2 + (1-b2)*(0*0)
    int32_t s = from + 2;
    for (; s <= t_done; ++s) {
      const float lr_s = lr_tab[s & kLrRingMask];
      bool moved = false;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        mm[q] = __fadd_rn(__fmul_rn(mm[q], b1), __fmul_rn(omb1, 0.f));
        vv[q] = __fadd_rn(__fmul_rn(vv[q], b2), __fmul_rn(omb2, 0.f));
        const float np = adam_move(pp[q], lr_s, mm[q], vv[q], eps, pos_eps);
        moved |= (__float_as_uint(np) != __float_as_uint(pp[q]));
        pp[q] = np;
      }
      if (rest_ok && !__any_sync(0xffffffffu, moved)) { ++s; break; }
    }
    for (; s <= t_done; ++s) {                    // theta rests: only the slots still decay
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        mm[q] = __fadd_rn(__fmul_rn(mm[q], b1), __fmul_rn(omb1, 0.f));
        vv[q] = __fadd_rn(__fmul_rn(vv[q], b2), __fmul_rn(omb2, 0.f));
      }
    }
    if (act) {
      *reinterpret_cast<float4*>(p + o) = P;
      *reinterpret_cast<float4*>(m + o) = M;
      *reinterpret_cast<float4*>(v + o) = V;
      if ((__float_as_uint(G.x) | __float_as_uint(G.y) | __float_as_uint(G.z) | __float_as_uint(G.w)) != 0u)
        *reinterpret_cast<float4*>(g + o) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// Catch-up of the rows a batch references.  Persistent grid: every warp scans 32 rows at a time (one coalesced
// read of their stamps and `last` values), then the whole warp walks the rows that need work.  So a row the
// batch references costs one pass (theta, m, v, g in; theta, m, v, 0 out) per step instead of a catch-up pass
// before the forward and an update pass after the backward.
// OCC = resident blocks per SM the kernel is compiled for; the persistent grid is launched as exactly one wave
// of num_sms * OCC blocks.
template <int MODE, int OCC>
__global__ void __launch_bounds__(256, OCC)
adam_rows_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, int rows, int d,
                 const int32_t* __restrict__ stamp, int32_t epoch, int32_t* __restrict__ last, int32_t t_done,
                 const float* __restrict__ lr_tab, float b1, float b2, float eps, int rest_ok, int pos_eps) {
  const int lane = threadIdx.x & 31;
  const int warp_global = (blockIdx.x * 256 + threadIdx.x) >> 5;
  const int total_warps = (gridDim.x * 256) >> 5;
  const float omb1 = __fsub_rn(1.f, b1), omb2 = __fsub_rn(1.f, b2);
  for (int base = warp_global * 32; base < rows; base += total_warps * 32) {
    const int r = base + lane;
    int32_t from_l = 0;
    bool hit = false;
    if (r < rows) {
      hit = (MODE == ADAM_ROWS_FLUSH) || (stamp[r] == epoch);
      if (hit) {
        from_l = last[r];
        if (from_l >= t_done) hit = false;
      }
    }
    unsigned todo = __ballot_sync(0xffffffffu, hit);
    auto prefetch_row = [&](int row) {           // the four 512-byte pieces of a row towards L2 while the previous row is replayed
      const size_t o = (size_t)row * d + lane * 4;
      if (lane * 4 < d) {
        asm volatile("prefetch.global.L2 [%0];" ::"l"(p + o));
        asm volatile("prefetch.global.L2 [%0];" ::"l"(m + o));
        asm volatile("prefetch.global.L2 [%0];" ::"l"(v + o));
        asm volatile("prefetch.global.L2 [%0];" ::"l"(g + o));
      }
    };
    if (todo) prefetch_row(base + __ffs(todo) - 1);
    while (todo) {
      const int b = __ffs(todo) - 1;
      todo &= todo - 1;
      if (todo) prefetch_row(base + __ffs(todo) - 1);
      const int32_t from = __shfl_sync(0xffffffffu, from_l, b);
      replay_row(p, g, m, v, (size_t)(base + b) * d, d, from, t_done, lr_tab, b1, b2, eps, omb1, omb2, lane, rest_ok != 0,
                 pos_eps != 0);
    }
    if (hit) last[r] = t_done;
  }
}

// Sweep / flush: EVERY row of [0, rows) that is behind is brought up to date, one warp per row (grid-stride), so
// a slice of a few ten thousand rows still spreads over every resident warp of the GPU.
template <int OCC>
__global__ void __launch_bounds__(256, OCC)
adam_sweep_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, int rows, int d,
                  int32_t* __restrict__ last, int32_t t_done, const float* __restrict__ lr_tab, float b1, float b2, float eps,
                  int rest_ok, int pos_eps) {
  const int lane = threadIdx.x & 31;
  const int warp_global = (blockIdx.x * 256 + threadIdx.x) >> 5;
  const int total_warps = (gridDim.x * 256) >> 5;
  const float omb1 = __fsub_rn(1.f, b1), omb2 = __fsub_rn(1.f, b2);
  for (int row = warp_global; row < rows; row += total_warps) {
    const int32_t from = last[row];
    if (from >= t_done) continue;
    replay_row(p, g, m, v, (size_t)row * d, d, from, t_done, lr_tab, b1, b2, eps, omb1, omb2, lane, rest_ok != 0, pos_eps != 0);
    __syncwarp();
    if (lane == 0) last[row] = t_done;
  }
}

// ---------------------------------------------------------------------------------------------
// Deterministic embedding-gradient reduction (option "deterministic", DESIGN.md section 5.1).
//
// The entries e = 3 n + seg of a batch are keyed by (table, row): key = row for the token table (seg 0, 2), T + row for the
// path table (seg 1), and nkeys = T + P for masked contexts, which therefore sort behind every real key and are never
// summed.  A stable LSD radix sort (8-bit digits: per-tile histograms, bucket_scan_kernel, stable per-tile scatter)
// lists each row's entries in increasing e.  A row's entries are then cut into chunks of kDetChunk, aligned at the row's
// first entry; each chunk is summed left to right from +0.0f by one warp, and the chunk sums of a row are added left to
// right from +0.0f.  The gradient row is zero before the step, so the sum is stored, not added.
// ---------------------------------------------------------------------------------------------
constexpr int kDetChunk = 32;                 // K: entries per chunk
constexpr int kDetSortThreads = 256;
constexpr int kDetSortTile = 4096;            // entries per radix-sort tile (16 rounds of 256)
constexpr int kDetRadix = 256;                // 8-bit digits

// key of entry e of a train step's batch
struct DetStepKeys {
  const int32_t* src;
  const int32_t* pth;
  const int32_t* tgt;
  const float* mask;
  int T;          // token rows: path keys start here
  uint32_t nkeys; // T + P: the key of a masked entry
  __device__ __forceinline__ uint32_t operator()(int e) const {
    const int n = e / 3, seg = e - 3 * n;
    if (mask[n] == 0.f) return nkeys;
    return seg == 1 ? (uint32_t)(T + pth[n]) : (uint32_t)(seg == 0 ? src[n] : tgt[n]);
  }
};
// key of entry e of c2v_selftest_row_sum: one row list of one table
struct DetListKeys {
  const int32_t* rows;
  int base;       // 0 (token table) or T (path table)
  __device__ __forceinline__ uint32_t operator()(int e) const { return (uint32_t)(base + rows[e]); }
};

template <class KeyFn>
__global__ void __launch_bounds__(256)
det_keys_kernel(const __grid_constant__ KeyFn key, int count, uint32_t* __restrict__ keys, int32_t* __restrict__ vals) {
  for (int e = blockIdx.x * 256 + threadIdx.x; e < count; e += gridDim.x * 256) {
    keys[e] = key(e);
    vals[e] = e;
  }
}

// hist[digit * tiles + tile] = entries of the tile whose key has this digit at `shift`
__global__ void __launch_bounds__(kDetSortThreads)
det_hist_kernel(const uint32_t* __restrict__ keys, int count, int shift, int32_t* __restrict__ hist) {
  __shared__ int32_t h[kDetRadix];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int lo = blockIdx.x * kDetSortTile, hi = min(count, lo + kDetSortTile);
  for (int i = lo + threadIdx.x; i < hi; i += kDetSortThreads) atomicAdd(&h[(keys[i] >> shift) & (kDetRadix - 1)], 1);
  __syncthreads();
  hist[threadIdx.x * gridDim.x + blockIdx.x] = h[threadIdx.x];
}

// Stable scatter of one tile: offs = exclusive scan of hist (digit-major), so the tile's entries with digit q go to
// offs[q * tiles + tile] onwards, in their order inside the tile.  The tile is walked in rounds of 256 entries; inside a
// round a warp ranks its lanes with __match_any_sync and the warps' counts are prefixed in warp order.
__global__ void __launch_bounds__(kDetSortThreads)
det_scatter_kernel(const uint32_t* __restrict__ keys, const int32_t* __restrict__ vals, int count, int shift,
                   const int32_t* __restrict__ offs, uint32_t* __restrict__ okeys, int32_t* __restrict__ ovals) {
  constexpr int W = kDetSortThreads / 32;
  __shared__ int32_t wc[W][kDetRadix];
  __shared__ int32_t run[kDetRadix];
  __shared__ int32_t goff[kDetRadix];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  run[tid] = 0;
  goff[tid] = offs[tid * gridDim.x + blockIdx.x];
  const int lo = blockIdx.x * kDetSortTile, hi = min(count, lo + kDetSortTile);
  for (int base = lo; base < hi; base += kDetSortThreads) {
#pragma unroll
    for (int w = 0; w < W; ++w) wc[w][tid] = 0;
    __syncthreads();
    const int i = base + tid;
    const bool valid = i < hi;
    const uint32_t k = valid ? keys[i] : 0u;
    const int q = valid ? (int)((k >> shift) & (kDetRadix - 1)) : kDetRadix + lane;      // idle lanes match nobody
    const unsigned peers = __match_any_sync(0xffffffffu, q);
    const int rank = __popc(peers & ((1u << lane) - 1u));
    if (valid && rank == 0) wc[warp][q] = __popc(peers);
    __syncthreads();
    {
      int r = run[tid];
#pragma unroll
      for (int w = 0; w < W; ++w) { const int c = wc[w][tid]; wc[w][tid] = r; r += c; }
      run[tid] = r;
    }
    __syncthreads();
    if (valid) {
      const int pos = goff[q] + wc[warp][q] + rank;
      okeys[pos] = k;
      ovals[pos] = vals[i];
    }
    __syncthreads();
  }
}

// contribution of entry e to columns [4 c4, 4 c4 + 4) of its row in a train step: dX'[n, seg d + col] x dropout multiplier x
// grad_scale, as scatter_dx_kernel (SIMT_ORDER false: g * (m * s)) or simt::ScatterDx (true: (g * m) * s) computes it
template <bool SIMT_ORDER>
struct DetStepContrib {
  const float* dX;
  Dropout dp;
  float grad_scale;
  int d;
  __device__ __forceinline__ float4 operator()(int e, int c4) const {
    const int n = e / 3, seg = e - 3 * n, j = seg * d + c4 * 4;
    float4 g = *reinterpret_cast<const float4*>(dX + (size_t)n * 3 * d + j);
    const float4 m = dropout_mult4(dp, n, j >> 2);
    if (SIMT_ORDER) {
      g.x = __fmul_rn(__fmul_rn(g.x, m.x), grad_scale); g.y = __fmul_rn(__fmul_rn(g.y, m.y), grad_scale);
      g.z = __fmul_rn(__fmul_rn(g.z, m.z), grad_scale); g.w = __fmul_rn(__fmul_rn(g.w, m.w), grad_scale);
    } else {
      g.x = __fmul_rn(g.x, __fmul_rn(m.x, grad_scale)); g.y = __fmul_rn(g.y, __fmul_rn(m.y, grad_scale));
      g.z = __fmul_rn(g.z, __fmul_rn(m.z, grad_scale)); g.w = __fmul_rn(g.w, __fmul_rn(m.w, grad_scale));
    }
    return g;
  }
};
// c2v_selftest_row_sum: entry e contributes vals[e, :]
struct DetListContrib {
  const float* vals;
  int d;
  __device__ __forceinline__ float4 operator()(int e, int c4) const {
    return *reinterpret_cast<const float4*>(vals + (size_t)e * d + c4 * 4);
  }
};

// Where the finished sum of key k's row goes (`first`: the sorted position of the row's first entry).
// DetDest: into the row itself -- token table for k < T, path table otherwise (the tables are local: one shard at most)
struct DetDest {
  float* tok;
  float* path;
  int T, d;
  __device__ __forceinline__ float* row(uint32_t k, int /*first*/) const {
    return (int)k < T ? tok + (size_t)k * d : path + (size_t)((int)k - T) * d;
  }
};

__device__ __forceinline__ float4 add4_rn(float4 a, const float4& b) {
  a.x = __fadd_rn(a.x, b.x); a.y = __fadd_rn(a.y, b.y); a.z = __fadd_rn(a.z, b.z); a.w = __fadd_rn(a.w, b.w);
  return a;
}

// slot of the partial of the chunk starting at sorted position i (first: it is its row's first chunk).  Rows with more
// than one chunk are longer than K, so a window [aK, aK + K) holds at most one first and one later chunk of such rows.
__device__ __forceinline__ size_t det_slot(int i, bool first) { return 2 * (size_t)(i / kDetChunk) + (first ? 1 : 0); }

// Pass 1: one warp per 32 sorted positions; every position that starts a chunk (its offset from its row's first entry is a
// multiple of K) is summed by the warp.  A row of one chunk is stored; otherwise the chunk sum goes to its partial slot.
template <class Contrib, class Dest>
__global__ void __launch_bounds__(256)
det_chunk_kernel(const uint32_t* __restrict__ keys, const int32_t* __restrict__ vals, int count, uint32_t nkeys,
                 const __grid_constant__ Contrib contrib, const __grid_constant__ Dest dst, float* __restrict__ part) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * 256 + threadIdx.x;
  bool start = false;
  int first = i;
  uint32_t k = nkeys;
  if (i < count) {
    k = keys[i];
    if (k < nkeys && i > 0 && keys[i - 1] == k) {        // inside a row: find the row's first entry (lower bound)
      int lo = 0, hi = i - 1;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (keys[mid] < k) lo = mid + 1; else hi = mid;
      }
      first = lo;
    }
    start = k < nkeys && (i - first) % kDetChunk == 0;
  }
  unsigned todo = __ballot_sync(0xffffffffu, start);
  const int d4 = dst.d / 4;
  while (todo) {
    const int b = __ffs(todo) - 1;
    todo &= todo - 1;
    const int p = __shfl_sync(0xffffffffu, i, b);
    const int f = __shfl_sync(0xffffffffu, first, b);
    const uint32_t kk = __shfl_sync(0xffffffffu, k, b);
    int end = p + 1;
    while (end < count && end < p + kDetChunk && keys[end] == kk) ++end;
    const bool single = p == f && !(end < count && keys[end] == kk);
    for (int c4 = lane; c4 < d4; c4 += 32) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int j = p; j < end; ++j) acc = add4_rn(acc, contrib(vals[j], c4));
      float* out = single ? dst.row(kk, f) : part + det_slot(p, p == f) * dst.d;
      reinterpret_cast<float4*>(out)[c4] = acc;
    }
  }
}

// Pass 2: the first position of every row with more than one chunk adds the row's chunk sums in order and stores the row.
template <class Dest>
__global__ void __launch_bounds__(256)
det_combine_kernel(const uint32_t* __restrict__ keys, int count, uint32_t nkeys, const __grid_constant__ Dest dst,
                   const float* __restrict__ part) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * 256 + threadIdx.x;
  bool lead = false;
  uint32_t k = nkeys;
  if (i < count) {
    k = keys[i];
    lead = k < nkeys && (i == 0 || keys[i - 1] != k) && i + kDetChunk < count && keys[i + kDetChunk] == k;
  }
  unsigned todo = __ballot_sync(0xffffffffu, lead);
  const int d4 = dst.d / 4;
  while (todo) {
    const int b = __ffs(todo) - 1;
    todo &= todo - 1;
    const int f = __shfl_sync(0xffffffffu, i, b);
    const uint32_t kk = __shfl_sync(0xffffffffu, k, b);
    float4* out = reinterpret_cast<float4*>(dst.row(kk, f));
    for (int c4 = lane; c4 < d4; c4 += 32) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int p = f; p < count && keys[p] == kk; p += kDetChunk)
        acc = add4_rn(acc, reinterpret_cast<const float4*>(part + det_slot(p, p == f) * dst.d)[c4]);
      out[c4] = acc;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Ordered gradient exchange for row-sharded tables (option "ordered_exchange", DESIGN.md section 5.1).
//
// Sender: the entries are keyed owner-major -- key = o L + (path table ? Tl + rho : rho) for global row r with owner
// o = r % W and local row rho = r / W, Tl / Pl rows per token / path shard, L = Tl + Pl; W L for masked contexts -- and
// sorted and reduced as above, so each distinct (owner, table, row) ends as ONE ordered sum.  The sums of owner o lie in key
// order, token rows before path rows: the k-th of them goes into slot k of this rank's region of o's inbox (the layout of
// the plain push: row ids, values, two counts per sender), where k is the row's head rank -- the exclusive scan of "sorted
// position starts a row" -- minus the head rank at o's first position.
// Owner: inbox_fold_ordered_kernel adds the senders' sums of a row in sender order and stores the row.
// ---------------------------------------------------------------------------------------------
struct ExchangeKeyMap {
  int shift, mask;     // as ShardedTable: owner = r & mask, local row = r >> shift
  int Tl, L;           // token rows per shard; token + path rows per shard
  __device__ __forceinline__ uint32_t key(int r, bool path) const {
    return (uint32_t)((r & mask) * L + (path ? Tl : 0) + (r >> shift));
  }
  __device__ __forceinline__ uint32_t nkeys() const { return (uint32_t)((mask + 1) * L); }
};
// key of entry e of a train step's batch
struct ExchangeStepKeys {
  const int32_t* src;
  const int32_t* pth;
  const int32_t* tgt;
  const float* mask;
  ExchangeKeyMap map;
  __device__ __forceinline__ uint32_t operator()(int e) const {
    const int n = e / 3, seg = e - 3 * n;
    if (mask[n] == 0.f) return map.nkeys();
    return map.key(seg == 0 ? src[n] : (seg == 1 ? pth[n] : tgt[n]), seg == 1);
  }
};
// key of entry e of c2v_selftest_exchange_push: n_tok global token rows, then global path rows
struct ExchangeListKeys {
  const int32_t* tok_rows;
  const int32_t* path_rows;
  int n_tok;
  ExchangeKeyMap map;
  __device__ __forceinline__ uint32_t operator()(int e) const {
    return e < n_tok ? map.key(tok_rows[e], false) : map.key(path_rows[e - n_tok], true);
  }
};

__device__ __forceinline__ bool det_is_head(const uint32_t* __restrict__ keys, int i, uint32_t nkeys) {
  const uint32_t k = keys[i];
  return k < nkeys && (i == 0 || keys[i - 1] != k);
}

// tile_heads[tile] = rows that start inside the tile of kDetSortTile sorted positions
__global__ void __launch_bounds__(kDetSortThreads)
det_head_count_kernel(const uint32_t* __restrict__ keys, int count, uint32_t nkeys, int32_t* __restrict__ tile_heads) {
  const int lo = blockIdx.x * kDetSortTile, hi = min(count, lo + kDetSortTile);
  int n = 0;
  for (int i = lo + threadIdx.x; i < hi; i += kDetSortThreads) n += det_is_head(keys, i, nkeys) ? 1 : 0;
  __shared__ int32_t total;
  if (threadIdx.x == 0) total = 0;
  __syncthreads();
  n = __reduce_add_sync(0xffffffffu, n);
  if ((threadIdx.x & 31) == 0 && n) atomicAdd(&total, n);
  __syncthreads();
  if (threadIdx.x == 0) tile_heads[blockIdx.x] = total;
}

// head_rank[i] = rows that start before sorted position i (tile_base = exclusive scan of tile_heads)
__global__ void __launch_bounds__(kDetSortThreads)
det_head_rank_kernel(const uint32_t* __restrict__ keys, int count, uint32_t nkeys, const int32_t* __restrict__ tile_base,
                     int32_t* __restrict__ head_rank) {
  constexpr int W = kDetSortThreads / 32;
  __shared__ int32_t wc[W];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int lo = blockIdx.x * kDetSortTile, hi = min(count, lo + kDetSortTile);
  int run = tile_base[blockIdx.x];
  for (int base = lo; base < hi; base += kDetSortThreads) {
    const int i = base + threadIdx.x;
    const bool head = i < hi && det_is_head(keys, i, nkeys);
    const unsigned heads = __ballot_sync(0xffffffffu, head);
    if (lane == 0) wc[warp] = __popc(heads);
    __syncthreads();
    int before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < W; ++w) { before += w < warp ? wc[w] : 0; all += wc[w]; }
    if (i < hi) head_rank[i] = run + before + __popc(heads & ((1u << lane) - 1u));
    run += all;
    __syncthreads();
  }
}

// rows that start before the first sorted position whose key is >= k
__device__ __forceinline__ int exchange_heads_below(const uint32_t* __restrict__ keys, const int32_t* __restrict__ head_rank,
                                                    int count, uint32_t nkeys, uint32_t k) {
  if (count == 0) return 0;
  int lo = 0, hi = count;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (keys[mid] < k) lo = mid + 1; else hi = mid;
  }
  if (lo < count) return head_rank[lo];
  return head_rank[count - 1] + (det_is_head(keys, count - 1, nkeys) ? 1 : 0);
}

// bounds[2 o] / bounds[2 o + 1] = head rank at the first token / path key of owner o, bounds[2 W] = distinct rows in all;
// the two counts of this sender go into every owner's inbox
__global__ void exchange_bounds_kernel(const uint32_t* __restrict__ keys, const int32_t* __restrict__ head_rank, int count,
                                       const __grid_constant__ ExchangeKeyMap map, const __grid_constant__ InboxSet inbox,
                                       int32_t* __restrict__ bounds) {
  __shared__ int32_t b[2 * kMaxShards + 1];
  const int j = threadIdx.x, W = map.mask + 1;
  if (j <= 2 * W) {
    b[j] = exchange_heads_below(keys, head_rank, count, map.nkeys(), (uint32_t)((j >> 1) * map.L + (j & 1) * map.Tl));
    bounds[j] = b[j];
  }
  __syncthreads();
  if (j < W) {
    InboxView v = inbox_of(inbox, j);
    v.cnt[2 * inbox.rank] = b[2 * j + 1] - b[2 * j];
    v.cnt[2 * inbox.rank + 1] = b[2 * j + 2] - b[2 * j + 1];
  }
}

// the inbox slot of key k's row, from the sorted position of the row's first entry
struct DetInboxDest {
  InboxSet inbox;
  const int32_t* head_rank;
  const int32_t* bounds;
  int L, d;
  __device__ __forceinline__ size_t slot(uint32_t k, int first) const {
    return (size_t)inbox.rank * inbox.cap + (size_t)(head_rank[first] - bounds[2 * (k / (uint32_t)L)]);
  }
  __device__ __forceinline__ float* row(uint32_t k, int first) const {
    return inbox_of(inbox, (int)(k / (uint32_t)L)).val + slot(k, first) * d;
  }
};

// ids[slot] = local row, for every row this sender pushes
__global__ void __launch_bounds__(256)
exchange_ids_kernel(const uint32_t* __restrict__ keys, int count, const __grid_constant__ ExchangeKeyMap map,
                    const __grid_constant__ DetInboxDest dst) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= count || !det_is_head(keys, i, map.nkeys())) return;
  const uint32_t k = keys[i];
  const int o = (int)(k / (uint32_t)map.L), rem = (int)(k - (uint32_t)o * map.L);
  inbox_of(dst.inbox, o).ids[dst.slot(k, i)] = rem < map.Tl ? rem : rem - map.Tl;
}

// position of `row` in the strictly increasing list ids[0, n), or -1
__device__ __forceinline__ int exchange_find(const int32_t* __restrict__ ids, int n, int row) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (ids[mid] < row) lo = mid + 1; else hi = mid;
  }
  return (lo < n && ids[lo] == row) ? lo : -1;
}

// The owner's half: one warp per (sender s, slot k) of this rank's inbox.  The warp of the lowest sender that lists a row
// leads it: from +0.0f it adds the row's sums of senders s, s + 1, ... in that order (each sender lists a row at most once,
// in increasing row order per table: binary search) and stores the row.  No atomics; persistent grid.
__global__ void __launch_bounds__(256)
inbox_fold_ordered_kernel(const __grid_constant__ InboxSet inbox, int d, float* __restrict__ g_tok, float* __restrict__ g_path) {
  const int lane = threadIdx.x & 31;
  const int warp_global = (blockIdx.x * 256 + threadIdx.x) >> 5, total_warps = (gridDim.x * 256) >> 5;
  const InboxView v = inbox_of(inbox, inbox.rank);
  for (int s = 0; s < inbox.world; ++s) {
    const int n_tok = v.cnt[2 * s], n_all = n_tok + v.cnt[2 * s + 1];
    for (int k = warp_global; k < n_all; k += total_warps) {
      const bool path = k >= n_tok;
      const int row = v.ids[(size_t)s * inbox.cap + k];
      // the list of the row's table in sender t's region: [begin, begin + n)
      auto find = [&](int t) {
        const int t_tok = v.cnt[2 * t];
        const size_t begin = (size_t)t * inbox.cap + (path ? t_tok : 0);
        const int q = exchange_find(v.ids + begin, path ? v.cnt[2 * t + 1] : t_tok, row);
        return q < 0 ? (size_t)-1 : begin + q;
      };
      bool lead = true;
      for (int t = 0; t < s && lead; ++t) lead = find(t) == (size_t)-1;
      if (!lead) continue;
      size_t at[kMaxShards];
#pragma unroll
      for (int t = 0; t < kMaxShards; ++t)
        at[t] = t == s ? (size_t)s * inbox.cap + k : ((t > s && t < inbox.world) ? find(t) : (size_t)-1);
      float* dst = (path ? g_path : g_tok) + (size_t)row * d;
      for (int j = lane * 4; j < d; j += 128) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int t = 0; t < kMaxShards; ++t)
          if (at[t] != (size_t)-1) acc = add4_rn(acc, *reinterpret_cast<const float4*>(v.val + at[t] * d + j));
        *reinterpret_cast<float4*>(dst + j) = acc;
      }
    }
  }
}

// Deterministic sampled-softmax target gradient.  The B + S row ids are read as one list L = (target[0..B), sampled[0..S));
// block j owns row L[j] if j is that row's first occurrence in L, and stores
//   sum over L in order: true terms dl[b,0] v_b (one product each), then sampled terms, each the chunk sums of
//   sampled_softmax_bwd_kernel (b in chunks of kSampledChunk, accumulated as there) added chunk by chunk
// -- every addition left to right from +0.0f.  The gradient rows are zero before the step (cleared or caught up).
__global__ void __launch_bounds__(kSampledThreads)
sampled_softmax_bwd_det_kernel(const float* __restrict__ v, const float* __restrict__ dl, const int32_t* __restrict__ target,
                               const int32_t* __restrict__ sampled, int B, int S, int D, float* __restrict__ g_tgt) {
  const int j = blockIdx.x;
  const int row = j < B ? target[j] : sampled[j - B];
  for (int q = 0; q < j; ++q)
    if ((q < B ? target[q] : sampled[q - B]) == row) return;          // not the first occurrence
  for (int i = threadIdx.x; i < D; i += kSampledThreads) {
    float acc = 0.f;
    for (int b = j < B ? j : B; b < B; ++b)
      if (target[b] == row) acc = __fadd_rn(acc, __fmul_rn(dl[(size_t)b * (S + 1)], v[(size_t)b * D + i]));
    for (int s = 0; s < S; ++s) {
      if (sampled[s] != row) continue;
      for (int b0 = 0; b0 < B; b0 += kSampledChunk) {
        const int b1 = min(B, b0 + kSampledChunk);
        float c = 0.f;
        for (int b = b0; b < b1; ++b) c += dl[(size_t)b * (S + 1) + 1 + s] * v[(size_t)b * D + i];
        acc = __fadd_rn(acc, c);
      }
    }
    g_tgt[(size_t)row * D + i] = acc;
  }
}

// ---------------------------------------------------------------------------------------------
// Sampled softmax on a row-sharded target table (fully sharded schedule, DESIGN.md section 6j): the rows move to the
// examples.  Every rank draws the same S negatives; the owners pack the negative rows and the rows of the Bt examples'
// targets into zero-filled buffers that one all-reduce / one reduce-scatter complete (each element has exactly one
// non-zero contributor); every rank runs the head of sampled_softmax_fwd_kernel on its own Bl examples against the
// compact rows, writes its partial target gradients, and after an all-gather the owners fold them in a fixed order.
// ---------------------------------------------------------------------------------------------

// Owner pack: row j of (neg_rows [S, D], true_rows [Bt, D]) = Ytab_local[id - row0] for id = sampled[j] resp. target[j]
// when this rank holds global row id (row0 <= id < row0 + Yl), else zeros.  D % 4 == 0, rows 16-byte aligned.
__global__ void __launch_bounds__(256)
sampled_pack_rows_kernel(const float* __restrict__ Ytab, int Yl, int row0, const int32_t* __restrict__ sampled, int S,
                         const int32_t* __restrict__ target, int Bt, int D, float* __restrict__ neg_rows,
                         float* __restrict__ true_rows) {
  const int D4 = D / 4;
  const size_t n = (size_t)(S + Bt) * D4;
  for (size_t k = (size_t)blockIdx.x * 256 + threadIdx.x; k < n; k += (size_t)gridDim.x * 256) {
    const int j = (int)(k / D4), c = (int)(k % D4);
    const int local = (j < S ? sampled[j] : target[j - S]) - row0;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (local >= 0 && local < Yl) x = reinterpret_cast<const float4*>(Ytab + (size_t)local * D)[c];
    float* dst = j < S ? neg_rows + (size_t)j * D : true_rows + (size_t)(j - S) * D;
    reinterpret_cast<float4*>(dst)[c] = x;
  }
}

// The head of sampled_softmax_fwd_kernel, operation for operation, with the rows read from the packed buffers: example b
// (of this rank's B) scores true_rows[b] (its target's row) and neg_rows[s] (sampled[s]'s row) instead of Ytab[target[b]]
// and Ytab[sampled[s]].  Writes loss_b [B], dl [B, 1+S] and dv [B, D].
__global__ void __launch_bounds__(kSampledThreads)
sampled_softmax_rows_fwd_kernel(const float* __restrict__ v, const float* __restrict__ true_rows,
                                const float* __restrict__ neg_rows, const int32_t* __restrict__ target,
                                const int32_t* __restrict__ sampled, int S, const float* __restrict__ logq_true,
                                const float* __restrict__ logq_samp, int D, float inv_batch, float* __restrict__ loss_b,
                                float* __restrict__ dl, float* __restrict__ dv) {
  extern __shared__ float sm[];
  float* vs = sm;                 // [D]
  float* lg = vs + D;             // [1 + S]
  __shared__ float red[32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int y = target[b];
  const float* yrow = true_rows + (size_t)b * D;
  for (int i = tid; i < D; i += kSampledThreads) vs[i] = v[(size_t)b * D + i];
  __syncthreads();
  for (int j = warp; j <= S; j += kSampledThreads / 32) {
    const float* r = (j == 0) ? yrow : neg_rows + (size_t)(j - 1) * D;
    float part = 0.f;
    for (int i = lane * 4; i < D; i += 128) {
      const float4 a = *reinterpret_cast<const float4*>(r + i);
      part += a.x * vs[i] + a.y * vs[i + 1] + a.z * vs[i + 2] + a.w * vs[i + 3];
    }
    part = warp_sum(part);
    if (lane == 0) {
      float l = part - ((j == 0) ? logq_true[b] : logq_samp[j - 1]);
      if (j > 0 && sampled[j - 1] == y) l = -1e9f;          // accidental hit
      lg[j] = l;
    }
  }
  __syncthreads();
  float m = -INFINITY;
  for (int j = tid; j <= S; j += kSampledThreads) m = fmaxf(m, lg[j]);
  m = block_max(m, red);
  float s = 0.f;
  for (int j = tid; j <= S; j += kSampledThreads) s += expf(lg[j] - m);
  s = block_sum(s, red);
  const float lse = m + logf(s);
  if (tid == 0) loss_b[b] = lse - lg[0];
  __syncthreads();
  for (int j = tid; j <= S; j += kSampledThreads) {
    float g = expf(lg[j] - lse);
    if (j == 0) g -= 1.f;
    g *= inv_batch;
    if (j > 0 && sampled[j - 1] == y) g = 0.f;
    lg[j] = g;
    dl[(size_t)b * (S + 1) + j] = g;
  }
  __syncthreads();
  for (int i = tid; i < D; i += kSampledThreads) {
    float acc = lg[0] * yrow[i];
    for (int j = 1; j <= S; ++j) acc += lg[j] * neg_rows[(size_t)(j - 1) * D + i];
    dv[(size_t)b * D + i] = acc;
  }
}

// One rank's true-row target gradient terms: g_true[b] = dl[b,0] v_b (one product each), one block per example.
__global__ void __launch_bounds__(kSampledThreads)
sampled_true_grad_kernel(const float* __restrict__ v, const float* __restrict__ dl, int S, int D, float* __restrict__ g_true) {
  const int b = blockIdx.x;
  const float g = dl[(size_t)b * (S + 1)];
  for (int i = threadIdx.x; i < D; i += kSampledThreads) g_true[(size_t)b * D + i] = __fmul_rn(g, v[(size_t)b * D + i]);
}

// One rank's negative-row target gradients: g_neg[s] = the sums over b of dl[b,1+s] v_b in chunks of kSampledChunk
// examples (each summed from 0 in b order, as sampled_softmax_bwd_det_kernel does), added chunk by chunk from +0.0f.
// Block (s, column tile of 32): its warps sum different chunks of the same 32 columns into shared memory, and warp 0
// adds them in chunk order, kNegGradRound chunks at a time -- so the S * D / 32 blocks fill the GPU even at small S and
// the serial loop per warp is B / kNegGradWarps examples.  No atomics: every element is written once.
constexpr int kNegGradWarps = 8;
constexpr int kNegGradRound = 64;
__global__ void __launch_bounds__(kNegGradWarps * 32)
sampled_neg_grad_kernel(const float* __restrict__ v, const float* __restrict__ dl, int B, int S, int D,
                        float* __restrict__ g_neg) {
  __shared__ float part[kNegGradRound][32];
  const int s = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i = blockIdx.y * 32 + lane;
  const int chunks = (B + kSampledChunk - 1) / kSampledChunk;
  float acc = 0.f;
  for (int q0 = 0; q0 < chunks; q0 += kNegGradRound) {
    const int nq = min(kNegGradRound, chunks - q0);
    for (int q = warp; q < nq; q += kNegGradWarps) {
      const int b0 = (q0 + q) * kSampledChunk, b1 = min(B, b0 + kSampledChunk);
      float c = 0.f;
      if (i < D)
        for (int b = b0; b < b1; ++b) c += dl[(size_t)b * (S + 1) + 1 + s] * v[(size_t)b * D + i];
      part[q][lane] = c;
    }
    __syncthreads();
    if (warp == 0)
      for (int q = 0; q < nq; ++q) acc = __fadd_rn(acc, part[q][lane]);
    __syncthreads();                                   // part is rewritten by the next round
  }
  if (warp == 0 && i < D) g_neg[(size_t)s * D + i] = acc;
}

// Owner fold of the partial target gradients.  The Bt + S row ids are read as one list L = (target[0..Bt), sampled[0..S));
// block j handles row L[j] if this rank holds it and j is its first occurrence in L, and stores into g_tgt (local rows)
//   from +0.0f, left to right: g_true[b] for every b (global example order) with target[b] == row, then for every s
//   (in s order) with sampled[s] == row, g_neg[r][s] for r = 0 .. world-1.
// Rows nobody references are not written (the caller clears the block first).  D <= kFoldThreads * kFoldCols.
constexpr int kFoldThreads = 256;
constexpr int kFoldCols = 4;
__global__ void __launch_bounds__(kFoldThreads)
sampled_target_fold_kernel(const float* __restrict__ g_true, const float* __restrict__ g_neg, int world,
                           const int32_t* __restrict__ target, int Bt, const int32_t* __restrict__ sampled, int S, int D,
                           int row0, int Yl, float* __restrict__ g_tgt) {
  __shared__ unsigned hits[kFoldThreads / 32];
  const int j = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int row = j < Bt ? target[j] : sampled[j - Bt];
  const int local = row - row0;
  if (local < 0 || local >= Yl) return;                              // another rank's row
  int dup = 0;
  for (int q = tid; q < j; q += kFoldThreads) dup |= (q < Bt ? target[q] : sampled[q - Bt]) == row;
  if (__syncthreads_or(dup)) return;                                 // not the first occurrence
  float acc[kFoldCols];
#pragma unroll
  for (int k = 0; k < kFoldCols; ++k) acc[k] = 0.f;
  // the matching entries of each tile of kFoldThreads, taken in index order
  auto fold_tile = [&](int base, bool hit, auto&& add) {
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) hits[warp] = m;
    __syncthreads();
    for (int w = 0; w < kFoldThreads / 32; ++w)
      for (unsigned bits = hits[w]; bits; bits &= bits - 1) add(base + w * 32 + __ffs(bits) - 1);
    __syncthreads();
  };
  for (int b0 = 0; b0 < Bt; b0 += kFoldThreads) {
    const int b = b0 + tid;
    fold_tile(b0, b < Bt && target[b] == row, [&](int e) {
#pragma unroll
      for (int k = 0; k < kFoldCols; ++k) {
        const int i = tid + k * kFoldThreads;
        if (i < D) acc[k] = __fadd_rn(acc[k], g_true[(size_t)e * D + i]);
      }
    });
  }
  for (int s0 = 0; s0 < S; s0 += kFoldThreads) {
    const int s = s0 + tid;
    fold_tile(s0, s < S && sampled[s] == row, [&](int e) {
      for (int r = 0; r < world; ++r) {
#pragma unroll
        for (int k = 0; k < kFoldCols; ++k) {
          const int i = tid + k * kFoldThreads;
          if (i < D) acc[k] = __fadd_rn(acc[k], g_neg[((size_t)r * S + e) * D + i]);
        }
      }
    });
  }
#pragma unroll
  for (int k = 0; k < kFoldCols; ++k) {
    const int i = tid + k * kFoldThreads;
    if (i < D) g_tgt[(size_t)local * D + i] = acc[k];
  }
}

// out[0] = parts[0] + parts[1] + ... + parts[n-1], left to right from +0.0f (one thread)
__global__ void sum_in_order_kernel(const float* __restrict__ parts, int n, float* __restrict__ out) {
  float acc = 0.f;
  for (int r = 0; r < n; ++r) acc = __fadd_rn(acc, parts[r]);
  out[0] = acc;
}

}  // namespace c2v
