// Hopper (sm_90a) tensor-core GEMM:  C[M,N] = A[M,K] . B[K,N],  fp32 storage, tf32 operands (10-bit
// mantissa), fp32 accumulation in registers  (C2V_MATH_TF32; C2V_MATH_3XTF32 issues three products).
//
// Persistent, warp-specialised, one CTA of four warpgroups per SM:
//   warpgroup 0     : producer -- fills a 4-stage shared-memory ring.  Operands arrive by TMA
//                     (cp.async.bulk.tensor, 128-byte swizzle, issued by one thread).  wgmma takes 32-bit
//                     (tf32) operands K-major only, so an MN-major operand lands as four 32 x 32 boxes that
//                     the four producer warps then transpose in place (transpose_box); the loads of the next
//                     steps stay in flight meanwhile.  An A-operand policy (AX*) may instead compute the A
//                     tile (softmax gradient of a logits tile, embedding gather).
//                     With B_T (the logits GEMM), warps 1-3 also write each B tile out transposed (store_b_transposed).
//   warpgroups 1, 2 : consumers -- each owns 64 rows of the 128-row tile and issues
//                     wgmma.mma_async m64n128k8 (tf32) into a 64-register accumulator per thread;
//                     then writes the accumulator to its shared-memory staging blocks and goes on to its
//                     next tile.
//   warpgroup 3     : epilogue -- drains each staged tile through the fused epilogue (store / tanh /
//                     log-sum-exp partials / split-K slice / Adam) while the consumers run the next tile's
//                     MMAs, so a tile costs the longer of the two rather than their sum.
// Every stage is published by an mbarrier (K-major TMA transaction bytes + one arrival per producer thread;
// MN-major boxes report to a second, per-stage "landed" barrier that the transposing warps wait on) and
// released by one arrival per consumer warp once the wgmma group that read it has retired.  The staging
// blocks are handed over by two more: epi_full (every consumer thread has written its accumulator) and
// epi_empty (every epilogue thread is done with the blocks).  setmaxnreg moves registers from the producer,
// which holds no accumulator, to the epilogue (not for the plain store, which does not need them).
// Out-of-range rows / K-tail are zero-filled (by TMA or by the loaders), so any M, N, K work; split-K
// over blockIdx-independent work items.  Every operand needs a 16-byte aligned base and a row pitch that is a
// multiple of 4 floats (operand_ok).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

#include "common.cuh"

namespace c2v {
namespace umma {

constexpr int BM = 128;          // rows of a tile: two consumer warpgroups x wgmma M = 64
constexpr int BN = 128;          // columns of a tile: wgmma N
constexpr int BK = 32;           // fp32 elements per stage along K = one 128-byte swizzle row
constexpr int WG_K = 8;          // K per wgmma for 32-bit operands (32 bytes)
constexpr int STAGES = 4;
constexpr int kThreads = 4 * 128;
// Registers per thread of each role.  The CTA starts with 128 per thread (64 K for 512 threads, the whole register
// file); the producer then gives some up to the epilogue, 1 x kRegsProducer + 2 x kRegsConsumer + 1 x kRegsEpilogue
// = 4 x 128, unless the epilogue functor sets kMoveRegs = false (EpiStore).
constexpr int kRegsProducer = 72;
constexpr int kRegsConsumer = 128;
constexpr int kRegsEpilogue = 184;
static_assert(kRegsProducer + 2 * kRegsConsumer + kRegsEpilogue == 4 * 128, "the roles share the CTA's registers");

// fast transcendental forms for the tensor-core path (operands are already tf32-rounded):
// exp via ex2.approx (rel. error 2^-22), tanh(x) = 1 - 2 / (exp(2x) + 1) (abs. error ~1e-7).
__device__ __forceinline__ float fast_tanh(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * 2.885390081777927f));      // exp(2x) = 2^(2 log2(e) x); +-inf / 0 at the ends are fine
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.f));
  return fmaf(-2.f, r, 1.f);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ---------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {      // no arrival
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// Bounded wait: a pipeline bug traps (reported as a CUDA error) instead of hanging the GPU.  SLEEP: between polls the
// warp sleeps, 32 ns at first and at most 256 ns -- for waits that can last a whole main loop (the epilogue warpgroup's
// on epi_full), so that the polling warps take no issue slots from the warps doing the work.
template <bool SLEEP = false>
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t ns = 32;
  while (!mbar_try_wait(bar, parity)) {
    if (SLEEP) {
      __nanosleep(ns);
      if (ns < 256) ns *= 2;
    }
    if (clock64() - t0 > 20000000000LL) __trap();     // ~10 s at 2 GHz
  }
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- TMA ----------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}

// ---- wgmma --------------------------------------------------------------------------------------
// Shared-memory matrix descriptor of a K-major SWIZZLE_128B tile (rows of 128 B, 16-byte chunk c of row r at
// (c ^ (r & 7)) * 16, 8-row groups 1024 B apart): start address >> 4 in [0,14), leading byte offset (unused
// for swizzled K-major layouts, 1) in [16,30), stride byte offset 1024 >> 4 in [32,46), swizzle mode 1 =
// 128B in [62,64).  The tile base is 1024-byte aligned; one wgmma consumes 32 B of each row, so the K step
// is +32 B on the start address.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// per-thread register budget of the executing warpgroup (all 128 threads): release / acquire down / up to R
template <int R>
__device__ __forceinline__ void wg_regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void wg_regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
// D[64 x 128] (+)= A[64 x 8] . B[8 x 128]; thread (warp w, lane l) holds rows 16w + l/4 (+8), columns 8j + 2(l%4) (+1)
// in d[4j + 2i + c] (row + 8i, column + c)
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
      "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate));
}

// ---- epilogues ---------------------------------------------------------------------------------------
// In the epilogue each thread holds one accumulator row's 32 consecutive columns at a time.  A
// functor supplies:  State / begin / end  -- per-(row, tile) state and its publication;
//                    observe(m, n0, 32 raw accumulators, nvalid, state) -- row-wise math (log-sum-exp);
//                    map(x)    -- the element-wise transform applied on the way out (identity, tanh);
//                    out(split), ldc -- where the tile goes;
//                    Pre / prefetch / store4 / store1(base, offset, value) -- what "storing" an element
//                    means (a plain write, or the optimizer update of the parameter the element is
//                    the gradient of; prefetch issues that update's loads ahead of the arithmetic).
// The store itself is done by store_chunk: registers (thread = row) -> a 4 KB XOR-swizzled
// shared-memory transpose per warp -> global stores in which every instruction writes four complete
// 128-byte row segments (storing straight from the row-per-thread layout would make each store
// instruction touch 32 different lines).
struct EpiNoState {};

struct EpiStore {
  using State = EpiNoState;
  float* C;
  size_t ldc;
  size_t split_stride;
  __device__ __forceinline__ void begin(State&) const {}
  __device__ __forceinline__ void end(int, int, int, bool, State&) const {}
  __device__ __forceinline__ void observe(int, int, const uint32_t (&)[32], int, State&) const {}
  __device__ __forceinline__ float map(float x) const { return x; }
  __device__ __forceinline__ float* out(int split) const { return C + (size_t)split * split_stride; }
  using Pre = EpiNoState;
  static constexpr int kRowBatch = 8;
  // A plain store needs no more than the 128 registers every role starts with; moving registers to the epilogue
  // warpgroup (setmaxnreg) made the long-K GEMM that uses this epilogue (dv: 743 K blocks per work item) 15 % slower.
  static constexpr bool kMoveRegs = false;
  __device__ __forceinline__ void prefetch(const float*, size_t, Pre&) const {}
  __device__ __forceinline__ void store4(float* c, size_t off, float4 v, const Pre&) const { *reinterpret_cast<float4*>(c + off) = v; }
  __device__ __forceinline__ void store1(float* c, size_t off, float x) const { c[off] = x; }
};
template <bool PRECISE>      // PRECISE: tanhf (the fp32-faithful 3xTF32 mode); else the ex2.approx form
struct EpiTanhStoreT {
  using State = EpiNoState;
  float* C;
  size_t ldc;
  __device__ __forceinline__ void begin(State&) const {}
  __device__ __forceinline__ void end(int, int, int, bool, State&) const {}
  __device__ __forceinline__ void observe(int, int, const uint32_t (&)[32], int, State&) const {}
  __device__ __forceinline__ float map(float x) const { return PRECISE ? tanhf(x) : fast_tanh(x); }
  __device__ __forceinline__ float* out(int) const { return C; }
  using Pre = EpiNoState;
  static constexpr int kRowBatch = 8;
  __device__ __forceinline__ void prefetch(const float*, size_t, Pre&) const {}
  __device__ __forceinline__ void store4(float* c, size_t off, float4 v, const Pre&) const { *reinterpret_cast<float4*>(c + off) = v; }
  __device__ __forceinline__ void store1(float* c, size_t off, float x) const { c[off] = x; }
};

// Logits epilogue: stores the tile of S and folds the row-wise (max, sum exp) of this warp's columns
// into a per-(row, partial slot) partial, so the cross entropy needs no extra pass over S for its
// log-sum-exp (tensorflow_model.py:227-230).
template <bool PRECISE>      // PRECISE: expf (3xTF32 mode); else ex2.approx
struct EpiStoreLseT {
  struct State { float mx, sum; };
  float* C;
  size_t ldc;
  float2* partial;       // [M, slots]; slot = 2 * n_tile + p, p = 0 for column quarters 0 and 2 of the tile, 1 for 1 and 3
  int slots;
  __device__ __forceinline__ float ex(float x) const { return PRECISE ? expf(x) : __expf(x); }
  __device__ __forceinline__ void begin(State& st) const { st.mx = -INFINITY; st.sum = 0.f; }
  __device__ __forceinline__ void end(int m, int slot, int, bool row_ok, State& st) const {
    if (row_ok) partial[(size_t)m * slots + slot] = make_float2(st.mx, st.sum);
  }
  __device__ __forceinline__ float map(float x) const { return x; }
  __device__ __forceinline__ float* out(int) const { return C; }
  using Pre = EpiNoState;
  static constexpr int kRowBatch = 8;
  __device__ __forceinline__ void prefetch(const float*, size_t, Pre&) const {}
  __device__ __forceinline__ void store4(float* c, size_t off, float4 v, const Pre&) const { *reinterpret_cast<float4*>(c + off) = v; }
  __device__ __forceinline__ void store1(float* c, size_t off, float x) const { c[off] = x; }
  __device__ __forceinline__ void observe(int, int, const uint32_t (&r)[32], int nvalid, State& st) const {
    float cm = -INFINITY;
    if (nvalid >= 32) {              // a full chunk (all but the last tile of a row): no per-element bounds
#pragma unroll
      for (int j = 0; j < 32; ++j) cm = fmaxf(cm, __uint_as_float(r[j]));
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j < nvalid) cm = fmaxf(cm, __uint_as_float(r[j]));
    }
    if (cm > st.mx) { st.sum *= ex(st.mx - cm); st.mx = cm; }
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    if (!PRECISE && nvalid >= 32) {
      // exp(x - mx) as one FFMA + one ex2.approx: 2^(x log2e - mx log2e)   (same 2^-22 relative accuracy as __expf)
      constexpr float L2E = 1.4426950408889634f;
      const float c = -st.mx * L2E;
      auto e2 = [](float t) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(t)); return y; };
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        a0 += e2(fmaf(__uint_as_float(r[j + 0]), L2E, c));
        a1 += e2(fmaf(__uint_as_float(r[j + 1]), L2E, c));
        a2 += e2(fmaf(__uint_as_float(r[j + 2]), L2E, c));
        a3 += e2(fmaf(__uint_as_float(r[j + 3]), L2E, c));
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        if (j + 0 < nvalid) a0 += ex(__uint_as_float(r[j + 0]) - st.mx);
        if (j + 1 < nvalid) a1 += ex(__uint_as_float(r[j + 1]) - st.mx);
        if (j + 2 < nvalid) a2 += ex(__uint_as_float(r[j + 2]) - st.mx);
        if (j + 3 < nvalid) a3 += ex(__uint_as_float(r[j + 3]) - st.mx);
      }
    }
    st.sum += (a0 + a1) + (a2 + a3);
  }
};

// Logits pass 1 of the recomputing schedule: ONLY the per-(row, partial slot) (max, sum exp) partials -- nothing is stored, so the
// epilogue neither transposes through shared memory nor writes the 1.07 GB slab (tensorflow_model.py:227-230).
template <bool PRECISE>
struct EpiLseOnlyT : EpiStoreLseT<PRECISE> {
  static constexpr bool kStores = false;
};
// Candidate epilogue of the row-sharded prediction (c2v_topk_partial): nothing is stored.  Each (row, partial slot) keeps
// the best k (value, column) pairs of its 64 columns in registers, value descending, ties to the lower column: an element
// enters only if it is strictly greater than the list's k-th value, the rule of topk_kernel, so NaN never enters and
// empty entries stay (-inf, INT_MAX).  A slot's columns arrive in increasing order (quarter p, then p + 2), which is what
// makes the strict rule put ties in index order.  end() writes the list to cand_val / cand_idx [M, slots, k] with global
// columns (local + row0).  LSE: the (max, sum exp) partials of EpiStoreLseT as well (normalize 2).
// The list is kTopkEpiMax registers long; for k < kTopkEpiMax its first kTopkEpiMax - k entries hold +inf, which no
// element passes, so the k-th value is always the last register.
constexpr int kTopkEpiMax = 16;
template <bool PRECISE, bool LSE>
struct EpiTopkT : EpiStoreLseT<PRECISE> {
  using Lse = EpiStoreLseT<PRECISE>;
  struct State {
    float v[kTopkEpiMax];
    int i[kTopkEpiMax];
    typename Lse::State ls;
  };
  float* cand_val;
  int32_t* cand_idx;
  int k;
  int row0;
  static constexpr bool kStores = false;
  __device__ __forceinline__ void begin(State& st) const {
#pragma unroll
    for (int q = 0; q < kTopkEpiMax; ++q) {
      st.v[q] = q < kTopkEpiMax - k ? INFINITY : -INFINITY;
      st.i[q] = INT_MAX;
    }
    if (LSE) Lse::begin(st.ls);
  }
  // x (column col) into the sorted list: c[q] = x > v[q] is monotone in q, so x lands before the first entry it beats and
  // the entries from there shift down one place; x <= v[K - 1] changes nothing.  Branch-free, so the 32 lanes run it in step.
  __device__ __forceinline__ void insert(float x, int col, State& st) const {
#pragma unroll
    for (int q = kTopkEpiMax - 1; q > 0; --q) {
      const bool here = x > st.v[q], above = x > st.v[q - 1];
      st.v[q] = above ? st.v[q - 1] : (here ? x : st.v[q]);
      st.i[q] = above ? st.i[q - 1] : (here ? col : st.i[q]);
    }
    if (x > st.v[0]) { st.v[0] = x; st.i[0] = col; }
  }
  // The chunk is screened against the list's k-th value as it stands (it only grows, so nothing screened out could
  // enter), then each lane inserts its survivors in column order: one rolled loop, so the epilogue's code stays small
  // enough for the instruction cache (fully unrolled, the 32 insertions made the kernel 35 K instructions long and the
  // product 7 times slower).  The loop reads the lane's next survivor at a per-lane index, which registers cannot serve:
  // from a copy of the chunk in local memory (128 bytes per thread, L1-resident).
  __device__ __forceinline__ void observe(int m, int n, const uint32_t (&r)[32], int nvalid, State& st) const {
    if (LSE) Lse::observe(m, n, r, nvalid, st.ls);
    const float kth = st.v[kTopkEpiMax - 1];
    float x[32];
    uint32_t todo = 0;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      x[j] = __uint_as_float(r[j]);
      if (j < nvalid && x[j] > kth) todo |= 1u << j;
    }
#pragma unroll 1
    while (todo) {
      const int j = __ffs(todo) - 1;
      todo &= todo - 1;
      insert(x[j], n + j, st);
    }
  }
  __device__ __forceinline__ void end(int m, int slot, int sp, bool row_ok, State& st) const {
    if (!row_ok) return;
    if (LSE) Lse::end(m, slot, sp, row_ok, st.ls);
    const size_t base = ((size_t)m * this->slots + slot) * k;
#pragma unroll
    for (int q = 0; q < kTopkEpiMax; ++q) {
      const int p = q - (kTopkEpiMax - k);
      if (p >= 0) {
        cand_val[base + p] = st.v[q];
        cand_idx[base + p] = st.i[q] == INT_MAX ? INT_MAX : st.i[q] + row0;
      }
    }
  }
};
// Logits pass 2: the same product again, and the epilogue writes dL/dlogits = (softmax - onehot) / B straight from the
// accumulator, given each row's log-sum-exp from pass 1: the slab is written once, as the gradient, and never read back
// by a softmax pass.  SPLIT (3xTF32): written as its tf32 split (high parts to C, residuals to C_lo).
template <bool PRECISE, bool SPLIT>
struct EpiSoftmaxGradT {
  struct State { float l; int tgt; };      // l: the row's log-sum-exp (PRECISE) or its exponent offset -lse log2e + log2(1/B)
  float* C;
  float* C_lo;
  size_t ldc;
  const float* lse;        // [M]
  const int32_t* target;   // [M] global class ids
  int row0;                // first class of this slab (row-sharded target table)
  float inv_batch;
  int M;
  __device__ __forceinline__ void begin(State& st) const { st.l = 0.f; st.tgt = -1; }
  __device__ __forceinline__ void end(int, int, int, bool, State&) const {}
  // called with this thread's row before any of its elements is mapped
  __device__ __forceinline__ void observe(int m, int, const uint32_t (&)[32], int, State& st) const {
    st.l = PRECISE ? lse[m] : fmaf(-lse[m], 1.4426950408889634f, log2f(inv_batch));
    st.tgt = target[m] - row0;
  }
  __device__ __forceinline__ float map(float x) const { return x; }
  __device__ __forceinline__ float map_at(float x, int col, const State& st) const {
    float p;
    if (PRECISE) {
      p = expf(x - st.l) * inv_batch;
    } else {          // exp(x - lse) / B as one FFMA + one ex2.approx
      asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(p) : "f"(fmaf(x, 1.4426950408889634f, st.l)));
    }
    return col == st.tgt ? p - inv_batch : p;
  }
  __device__ __forceinline__ float* out(int) const { return C; }
  using Pre = EpiNoState;
  static constexpr int kRowBatch = 8;
  __device__ __forceinline__ void prefetch(const float*, size_t, Pre&) const {}
  __device__ __forceinline__ void store4(float* c, size_t off, float4 v, const Pre&) const {
    if (SPLIT) {
      float4 hi, lo;
      split_tf32(v, hi, lo);
      *reinterpret_cast<float4*>(c + off) = hi;
      *reinterpret_cast<float4*>(C_lo + off) = lo;
    } else {
      *reinterpret_cast<float4*>(c + off) = v;
    }
  }
  __device__ __forceinline__ void store1(float* c, size_t off, float x) const {
    if (SPLIT) {
      float hi, lo;
      split_tf32(x, hi, lo);
      c[off] = hi; C_lo[off] = lo;
    } else {
      c[off] = x;
    }
  }
};

// Logits epilogue of the deferred-normalisation schedule (option "exp_slab"): the slab receives U = exp(s - c_row) instead
// of the logits, c_row a per-example constant known before the product (the example's true-class logit), and the partial of
// each (row, slot) holds (max U, sum U).  softmax - onehot is then U with one patched element per row times a per-row
// factor 1 / sum U, which the two gradient GEMMs apply to their small operand / result: no pass ever reads the slab back
// to normalise it (tensorflow_model.py:227-230).  max U is the range guard: the caller falls back to the two-pass
// schedule when some row's largest U leaves [kExpSlabMin, kExpSlabMax] (common.cuh).  SPLIT (3xTF32): U is written as its tf32 split.
template <bool PRECISE, bool SPLIT>
struct EpiExpSumT {
  struct State { float mx, sum; };
  float* C;
  float* C_lo;
  size_t ldc;
  const float* offset;   // [M] c_row
  float2* partial;       // [M, slots]; slot = 2 * n_tile + p, p = 0 for column quarters 0 and 2 of the tile, 1 for 1 and 3
  int slots;
  __device__ __forceinline__ void begin(State& st) const { st.mx = 0.f; st.sum = 0.f; }
  __device__ __forceinline__ void end(int m, int slot, int, bool row_ok, State& st) const {
    if (row_ok) partial[(size_t)m * slots + slot] = make_float2(st.mx, st.sum);
  }
  __device__ __forceinline__ float map(float x) const { return x; }
  __device__ __forceinline__ float* out(int) const { return C; }
  using Pre = EpiNoState;
  static constexpr int kRowBatch = 8;
  __device__ __forceinline__ void prefetch(const float*, size_t, Pre&) const {}
  __device__ __forceinline__ void store4(float* c, size_t off, float4 v, const Pre&) const {
    if (SPLIT) {
      float4 hi, lo;
      split_tf32(v, hi, lo);
      *reinterpret_cast<float4*>(c + off) = hi;
      *reinterpret_cast<float4*>(C_lo + off) = lo;
    } else {
      *reinterpret_cast<float4*>(c + off) = v;
    }
  }
  __device__ __forceinline__ void store1(float* c, size_t off, float x) const {
    if (SPLIT) {
      float hi, lo;
      split_tf32(x, hi, lo);
      c[off] = hi; C_lo[off] = lo;
    } else {
      c[off] = x;
    }
  }
  // rewrites the chunk's accumulators IN PLACE (the store that follows maps with the identity)
  __device__ __forceinline__ void observe(int m, int, uint32_t (&r)[32], int nvalid, State& st) const {
    const float c = offset[m];
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, x0 = 0.f, x1 = 0.f, x2 = 0.f, x3 = 0.f;
    if (!PRECISE && nvalid >= 32) {
      constexpr float L2E = 1.4426950408889634f;
      const float c2 = -c * L2E;           // exp(x - c) as one FFMA + one ex2.approx
      auto e2 = [](float t) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(t)); return y; };
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const float u0 = e2(fmaf(__uint_as_float(r[j + 0]), L2E, c2)), u1 = e2(fmaf(__uint_as_float(r[j + 1]), L2E, c2));
        const float u2 = e2(fmaf(__uint_as_float(r[j + 2]), L2E, c2)), u3 = e2(fmaf(__uint_as_float(r[j + 3]), L2E, c2));
        r[j + 0] = __float_as_uint(u0); r[j + 1] = __float_as_uint(u1); r[j + 2] = __float_as_uint(u2); r[j + 3] = __float_as_uint(u3);
        a0 += u0; a1 += u1; a2 += u2; a3 += u3;
        x0 = fmaxf(x0, u0); x1 = fmaxf(x1, u1); x2 = fmaxf(x2, u2); x3 = fmaxf(x3, u3);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        float u = 0.f;
        if (j < nvalid) u = PRECISE ? expf(__uint_as_float(r[j]) - c) : __expf(__uint_as_float(r[j]) - c);
        r[j] = __float_as_uint(u);
        if ((j & 3) == 0) { a0 += u; x0 = fmaxf(x0, u); }
        else if ((j & 3) == 1) { a1 += u; x1 = fmaxf(x1, u); }
        else if ((j & 3) == 2) { a2 += u; x2 = fmaxf(x2, u); }
        else { a3 += u; x3 = fmaxf(x3, u); }
      }
    }
    st.sum += (a0 + a1) + (a2 + a3);
    st.mx = fmaxf(st.mx, fmaxf(fmaxf(x0, x1), fmaxf(x2, x3)));
  }
};
// The two-pass fallback of that schedule is launched every step behind a device-side gate: a logits epilogue that carries
// `gate` makes the whole kernel return at once while *gate == 0.
template <bool PRECISE>
struct EpiStoreLseGatedT : EpiStoreLseT<PRECISE> {
  const int* gate;
};

using EpiTanhStore = EpiTanhStoreT<false>;
using EpiTanhStorePrecise = EpiTanhStoreT<true>;
using EpiStoreLse = EpiStoreLseT<false>;
using EpiStoreLsePrecise = EpiStoreLseT<true>;

// Target-table gradient epilogue with the optimizer folded in (option "fuse_target_adam"): the
// accumulator element is dYtab[y, j]; instead of writing it out for adam_kernel to read back, the
// epilogue applies TF1 Adam (SURVEY A.3, tensorflow_model.py:232) to (theta, m, v) in place -- the
// same correctly rounded fp32 operations in the same order as adam_kernel, so the result is
// bit-identical; the gradient itself is never stored.
struct EpiAdam {
  using State = EpiNoState;
  float* P;          // theta [M, ldc]; m and v have the same layout
  float* Mo;
  float* Vo;
  size_t ldc;
  float lr_t, b1, b2, eps, omb1, omb2;
  int l2_prefetch;   // engine option "adam_epilogue_prefetch"
  __device__ __forceinline__ void begin(State&) const {}
  __device__ __forceinline__ void end(int, int, int, bool, State&) const {}
  __device__ __forceinline__ void observe(int, int, const uint32_t (&)[32], int, State&) const {}
  __device__ __forceinline__ float map(float x) const { return x; }
  __device__ __forceinline__ float* out(int) const { return P; }
  __device__ __forceinline__ void upd(float& pp, float gg, float& mm, float& vv) const {
    mm = __fadd_rn(__fmul_rn(mm, b1), __fmul_rn(omb1, gg));
    vv = __fadd_rn(__fmul_rn(vv, b2), __fmul_rn(omb2, __fmul_rn(gg, gg)));
    pp = adam_move_dense(pp, lr_t, mm, vv, eps);
  }
  // Called by an epilogue thread one tile AHEAD of the tile it is about to drain (row m, columns [n0, n0 + ncols)): pulls the
  // (theta, m, v) lines of that region into L2, so that the update's loads -- only kRowBatch rows of them in flight per
  // thread -- see L2 latency rather than DRAM latency.
  __device__ __forceinline__ void prefetch_tile(int m, int n0, int ncols, int M, int N) const {
    if (m >= M || !l2_prefetch) return;
    const size_t row = (size_t)m * ldc;
    for (int n = n0; n < n0 + ncols && n < N; n += 32) {
      asm volatile("prefetch.global.L2 [%0];" ::"l"(P + row + n));
      asm volatile("prefetch.global.L2 [%0];" ::"l"(Mo + row + n));
      asm volatile("prefetch.global.L2 [%0];" ::"l"(Vo + row + n));
    }
  }
  struct Pre { float4 p, m, v; };
  // rows whose (theta, m, v) loads are in flight together per thread; the epilogue warpgroup's kRegsEpilogue registers
  // hold them without spilling
  static constexpr int kRowBatch = 4;
  __device__ __forceinline__ void prefetch(const float* c, size_t off, Pre& q) const {
    q.p = *reinterpret_cast<const float4*>(c + off);
    q.m = *reinterpret_cast<const float4*>(Mo + off);
    q.v = *reinterpret_cast<const float4*>(Vo + off);
  }
  __device__ __forceinline__ void store4(float* c, size_t off, float4 g, const Pre& q) const {
    float4 p = q.p, m = q.m, v = q.v;
    upd(p.x, g.x, m.x, v.x); upd(p.y, g.y, m.y, v.y); upd(p.z, g.z, m.z, v.z); upd(p.w, g.w, m.w, v.w);
    *reinterpret_cast<float4*>(c + off) = p;
    *reinterpret_cast<float4*>(Mo + off) = m;
    *reinterpret_cast<float4*>(Vo + off) = v;
  }
  __device__ __forceinline__ void store1(float* c, size_t off, float g) const {
    float p = c[off], m = Mo[off], v = Vo[off];
    upd(p, g, m, v);
    c[off] = p; Mo[off] = m; Vo[off] = v;
  }
};

// One 32-column chunk: registers (thread = row) -> swizzled smem -> coalesced global stores.
// element-wise transform on the way out: functors with a (row, column)-dependent transform define map_at(x, column, state)
template <class Epi>
__device__ __forceinline__ auto epi_map(const Epi& epi, float x, int col, const typename Epi::State& st, int)
    -> decltype(epi.map_at(x, col, st)) {
  return epi.map_at(x, col, st);
}
template <class Epi>
__device__ __forceinline__ float epi_map(const Epi& epi, float x, int, const typename Epi::State&, long) {
  return epi.map(x);
}
template <class Epi>
__device__ __forceinline__ auto epi_gate_closed(const Epi& epi, int) -> decltype(*epi.gate == 0) { return *epi.gate == 0; }
template <class Epi>
__device__ __forceinline__ bool epi_gate_closed(const Epi&, long) { return false; }
template <class Epi>
__device__ __forceinline__ auto epi_prefetch_tile(const Epi& epi, int m, int n0, int ncols, int M, int N, int)
    -> decltype(epi.prefetch_tile(m, n0, ncols, M, N)) {
  epi.prefetch_tile(m, n0, ncols, M, N);
}
template <class Epi>
__device__ __forceinline__ void epi_prefetch_tile(const Epi&, int, int, int, int, int, long) {}
template <class Epi>
constexpr bool epi_move_regs(...) { return true; }
template <class Epi, bool V = Epi::kMoveRegs>
constexpr bool epi_move_regs(int) { return V; }
template <class Epi>
constexpr bool epi_stores(...) { return true; }
template <class Epi, bool V = Epi::kStores>
constexpr bool epi_stores(int) { return V; }

template <class Epi>
__device__ __forceinline__ void store_chunk(const Epi& epi, const typename Epi::State& est, const uint32_t (&r)[32], float* stage, int lane,
                                            int m_base, int n, int M, int N, float* cbase, size_t ldc) {
#pragma unroll
  for (int j4 = 0; j4 < 8; ++j4) {
    const int pos = j4 ^ (lane & 7);
    *reinterpret_cast<float4*>(stage + lane * 32 + pos * 4) =
        make_float4(epi_map(epi, __uint_as_float(r[4 * j4]), n + 4 * j4, est, 0), epi_map(epi, __uint_as_float(r[4 * j4 + 1]), n + 4 * j4 + 1, est, 0),
                    epi_map(epi, __uint_as_float(r[4 * j4 + 2]), n + 4 * j4 + 2, est, 0), epi_map(epi, __uint_as_float(r[4 * j4 + 3]), n + 4 * j4 + 3, est, 0));
  }
  __syncwarp();
  const int col4 = lane & 7;
  const int gn = n + col4 * 4;
  // two passes per batch of rows so that a read-modify-write epilogue has kBatch rows' loads in flight
  constexpr int kBatch = Epi::kRowBatch;
  static_assert(8 % kBatch == 0, "the batches tile the chunk's 8 row groups: a remainder would reach into the next block");
#pragma unroll
  for (int it0 = 0; it0 < 8; it0 += kBatch) {
    float4 v[kBatch];
    typename Epi::Pre pre[kBatch];
#pragma unroll
    for (int i = 0; i < kBatch; ++i) {
      const int row = (it0 + i) * 4 + (lane >> 3);
      v[i] = *reinterpret_cast<const float4*>(stage + row * 32 + ((col4 ^ (row & 7)) * 4));
      const int gm = m_base + row;
      if (gm < M && gn + 3 < N) epi.prefetch(cbase, (size_t)gm * ldc + gn, pre[i]);
    }
#pragma unroll
    for (int i = 0; i < kBatch; ++i) {
      const int gm = m_base + (it0 + i) * 4 + (lane >> 3);
      if (gm < M && gn < N) {
        const size_t off = (size_t)gm * ldc + gn;
        if (gn + 3 < N) {
          epi.store4(cbase, off, v[i], pre[i]);
        } else {
          epi.store1(cbase, off, v[i].x);
          if (gn + 1 < N) epi.store1(cbase, off + 1, v[i].y);
          if (gn + 2 < N) epi.store1(cbase, off + 2, v[i].z);
        }
      }
    }
  }
  __syncwarp();
}

// ---- A-operand policies -------------------------------------------------------------------------------------
// Where the producer warpgroup gets the A tile from:
//   AXNone        : the A operand (TMA; MN-major tiles are then transposed in shared memory)
//   AXSoftmaxGrad : the A operand is a LOGITS slab S; the loaders turn each element into dL/dlogits =
//                   (softmax(S) - onehot) / B on its way into shared memory, given the per-row log-sum-exp,
//                   so that the separate pass that rewrote the slab (read + write) disappears (option
//                   fuse_softmax_grad):
//                     dv = P . Ytab     A = S, K-major   (rows = examples, K = classes)  -> AXSoftmaxGrad<true>
//                     dY = P^T . v      A = S^T, MN-major (rows = classes, K = examples) -> AXSoftmaxGrad<false>
//   AXGather      : the A tile is gathered from the embedding tables (fused context forward, see launch_ctx_fused)
struct AXNone {
  static constexpr int kKind = 0;
};

struct SoftmaxGradArgs {
  const float* lse;          // [examples] log-sum-exp of each row of S (all classes, all ranks)
  const int32_t* target;     // [examples] true class (global id)
  int row0;                  // first class held in S (row-sharded target table), 0 otherwise
  float inv_batch;
};
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
constexpr float kLog2e = 1.4426950408889634f;

template <bool EX_IS_M>      // true: tile rows are examples (A = S, K-major); false: tile K is examples (A = S^T, MN-major)
struct AXSoftmaxGrad {
  static constexpr int kKind = 1;
  SoftmaxGradArgs a;
  // p = exp(s - lse) / B as one fused multiply-add and one ex2: 2^(s log2(e) + c), c = -lse log2(e) + log2(1/B);
  // example ex's c and true class (relative to row0):
  __device__ __forceinline__ void example(int ex, float& c, int& tgt) const {
    c = fmaf(-a.lse[ex], kLog2e, log2f(a.inv_batch));
    tgt = a.target[ex] - a.row0;
  }
  // element s = S(ex, y) of an example with (c, tgt)
  __device__ __forceinline__ float p(float s, int y, float c, int tgt) const {
    return ex2_approx(fmaf(s, kLog2e, c)) - ((y == tgt) ? a.inv_batch : 0.f);
  }
  // K-major: v = A(x, k .. k+3), the four elements share example x.  Elements outside [X, K) are zero fill and stay zero.
  __device__ __forceinline__ float4 xform(float4 v, int x, int k, int X, int K) const {
    static_assert(EX_IS_M, "the MN-major tile is transformed element by element as it is transposed (umma_gemm_kernel)");
    if (x >= X) return v;
    float c;
    int tgt;
    example(x, c, tgt);
    float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) e[j] = (k + j < K) ? p(e[j], k + j, c, tgt) : 0.f;
    return make_float4(e[0], e[1], e[2], e[3]);
  }
};

struct AXGather {
  static constexpr int kKind = 2;
  ContextSource cs;
  Dropout dp;
  float* Xout;               // nullptr, or [M, 3d]: the dropped-out rows are written once (for dW = X'^T . dU)
};

// ---- tile loaders (producer warpgroup, thread t in [0, 128)) -----------------------------------------------------
__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// K-major operand (element (x, k) at base[x * ld + k]), rows x0 .. x0+127, k0 .. k0+31 -> SWIZZLE_128B tile.
// Thread t owns 16-byte chunk c = t % 8 of rows t / 8 + 16 i.
template <class AX>
__device__ __forceinline__ void load_tile_k(uint8_t* dst, const float* base, size_t ld, int x0, int X, int k0, int K, int t,
                                            const AX& ax) {
  const int c = t & 7, rg = t >> 3, k = k0 + c * 4;
  float4 v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int x = x0 + rg + 16 * i;
    v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (x < X) {
      const float* p = base + (size_t)x * ld + k;
      if (k + 3 < K) {
        v[i] = ld4(p);
      } else {
        if (k < K) v[i].x = p[0];
        if (k + 1 < K) v[i].y = p[1];
        if (k + 2 < K) v[i].z = p[2];
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = rg + 16 * i;
    if constexpr (AX::kKind == 1) v[i] = ax.xform(v[i], x0 + r, k, X, K);
    *reinterpret_cast<float4*>(dst + r * 128 + ((c ^ (r & 7)) << 4)) = v[i];
  }
}

// MN-major operand (element (x, k) at base[k * ld + x]), same tile.  TMA brings it in as four boxes: box q holds
// x0 + 32q .. +31 for the stage's 32 k, as 32 swizzled 128-byte rows (k) of 32 x, at bytes 4096q .. of the tile --
// the bytes that rows 32q .. 32q+31 of the K-major tile occupy.  So each warp rewrites one box in place: lane l
// reads column x = 32q + l, one element per k-row (a warp reads one 128-byte row at a time: no bank conflict),
// f(s, k) maps each element on the way, and the lane writes its tile row as 8 swizzled float4 chunks (each 8-lane
// store phase covers 8 distinct 16-byte bank groups).  TMA's zero fill of out-of-range x and k carries over.
// The box is 1024-byte aligned, so the swizzle is an XOR on one per-lane base address (element (l, k) at
// (box + 4l) ^ ((k & 7) << 4) + 128k, chunk c of row l at (box + 128l) ^ ((l & 7) << 4) ^ (c << 4)): written so, as
// shared-memory instructions, the addresses cost one XOR each instead of 40 loop-invariant registers.
template <class F>
__device__ __forceinline__ void transpose_box(uint8_t* box, int lane, const F& f) {
  const uint32_t rd = smem_u32(box) + lane * 4, wr = (smem_u32(box) + lane * 128) ^ ((lane & 7) << 4);
  float v[BK];
#pragma unroll
  for (int k = 0; k < BK; ++k) {
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v[k]) : "r"((rd ^ ((k & 7) << 4)) + k * 128) : "memory");
    v[k] = f(v[k], k);
  }
  __syncwarp();
#pragma unroll
  for (int c = 0; c < BK / 4; ++c)
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(wr ^ (c << 4)), "f"(v[4 * c]), "f"(v[4 * c + 1]), "f"(v[4 * c + 2]),
                 "f"(v[4 * c + 3]) : "memory");
}

// Where a GEMM with B_T writes its B operand's K-major transpose [K, ld] (element (n, k) at hi[k * ld + n]; 3xTF32: the
// transposed high parts to hi and the residuals to lo): the logits GEMM makes Ytab^T for dv from the Ytab tiles it streams
// anyway, instead of a separate pass that reads the table again.
struct BTransposed {
  float* hi;
  float* lo;
  size_t ld;
};

// The B tile of a full stage (rows n0 .. n0+127, k0 .. k0+31; chunk c of row r at (c ^ (r & 7)) * 16) to dst[k * ld + n] for
// n < N, k < K (K % 4 == 0: a chunk lies wholly inside K or outside it).  Copying warp cw in [0, 3) takes chunks cw, cw + 3,
// ...; lane l rows 4l .. 4l+3, so each of a chunk's four float4 stores writes 512 consecutive bytes of one row of dst.  At
// step j lane l reads row 4l + (j ^ s), s = (l >> 1) & 3: the 8 lanes of a quarter-warp then read rows that differ in
// (r & 7), i.e. 8 distinct 16-byte bank groups, and two conditional swaps put the four rows back in order.  The stores
// stream (evict-first): dst is read by a later GEMM, and L2 is better spent on the B tiles the other m-tiles still read.
__device__ __forceinline__ void store_b_transposed(const uint8_t* sb, float* dst, size_t ld, int n0, int N, int k0, int K, int cw,
                                                   int lane) {
  const int s = (lane >> 1) & 3, n = n0 + 4 * lane;
#pragma unroll 1
  for (int c = cw; c < BK / 4 && k0 + 4 * c < K; c += 3) {
    float4 v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = 4 * lane + (j ^ s);
      v[j] = *reinterpret_cast<const float4*>(sb + r * 128 + ((c ^ (r & 7)) << 4));
    }
    if (s & 1) { const float4 t0 = v[0], t2 = v[2]; v[0] = v[1]; v[1] = t0; v[2] = v[3]; v[3] = t2; }
    if (s & 2) { const float4 t0 = v[0], t1 = v[1]; v[0] = v[2]; v[1] = v[3]; v[2] = t0; v[3] = t1; }
    const float4 o[4] = {make_float4(v[0].x, v[1].x, v[2].x, v[3].x), make_float4(v[0].y, v[1].y, v[2].y, v[3].y),
                         make_float4(v[0].z, v[1].z, v[2].z, v[3].z), make_float4(v[0].w, v[1].w, v[2].w, v[3].w)};
    float* p = dst + (size_t)(k0 + 4 * c) * ld + n;
#pragma unroll
    for (int i = 0; i < 4; ++i, p += ld) {
      if (n + 3 < N) {
        __stcs(reinterpret_cast<float4*>(p), o[i]);
      } else {          // the last n-tile: columns n >= N are TMA's zero fill, and dst's padding there stays as it is
        if (n < N) __stcs(p, o[i].x);
        if (n + 1 < N) __stcs(p + 1, o[i].y);
        if (n + 2 < N) __stcs(p + 2, o[i].z);
      }
    }
  }
}

// gather(cs)[m0 .. m0+127, k-block kb] with dropout, as load_tile_k lays it out (d % 32 == 0: a k-block lies in one
// of the three segments source token | path | target token)
__device__ __forceinline__ void load_tile_gather(uint8_t* dst, const AXGather& g, int m0, int M, int kb, bool write_x, int t) {
  const int c = t & 7, rg = t >> 3;
  const int kps = g.cs.d / BK, seg = kb / kps;
  const int col = (kb - seg * kps) * BK + c * 4;
  const int32_t* ids = seg == 0 ? g.cs.src : seg == 1 ? g.cs.pth : g.cs.tgt;
  const int K = 3 * g.cs.d;
  float4 v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + rg + 16 * i;
    v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m < M) v[i] = ld4(((seg == 1) ? table_row(g.cs.path, ids[m], g.cs.d) : table_row(g.cs.tok, ids[m], g.cs.d)) + col);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = rg + 16 * i, m = m0 + r;
    if (g.dp.enabled) {
      const float4 mlt = dropout_mult4(g.dp, m, kb * (BK / 4) + c);
      v[i].x *= mlt.x; v[i].y *= mlt.y; v[i].z *= mlt.z; v[i].w *= mlt.w;
    }
    *reinterpret_cast<float4*>(dst + r * 128 + ((c ^ (r & 7)) << 4)) = v[i];
    if (write_x && m < M) *reinterpret_cast<float4*>(g.Xout + (size_t)m * K + kb * BK + c * 4) = v[i];
  }
}

// ---- kernel -------------------------------------------------------------------------------------------
struct GemmShape {
  int M, N, K;
  int m_tiles, n_tiles, splits;
  int kblocks_per_split;      // K blocks (of BK) per split-K slice
  int n_fastest;              // raster order of work items: 1 = consecutive items share the A tile
  int terms;                  // 1 = plain tf32;  3 = 3xTF32: every K block is issued as A_lo.B_hi + A_hi.B_lo + A_hi.B_hi
};
// the A operand as a raw pointer, for the one loader that does not go through TMA (load_tile_k: AXSoftmaxGrad<true>)
struct GemmPtrs {
  const float* a;
  size_t lda;
};

struct SmemLayout {
  static constexpr int kABytes = BM * BK * 4;          // 16 KB
  static constexpr int kBBytes = BN * BK * 4;          // 16 KB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kEpiOffset = STAGES * kStageBytes;                     // per consumer warpgroup: 64 x BN fp32
  static constexpr int kEpiBytes = 64 * BN * 4;
  static constexpr int kBarOffset = kEpiOffset + 2 * kEpiBytes;
  // barriers (full, empty, landed per stage; epi_full, epi_empty), + slack for 1024-B alignment
  static constexpr int kTotal = kBarOffset + 256 + 1024;
  static_assert((3 * STAGES + 2) * 8 <= 256, "the barriers fit their block");
  static_assert(kTotal <= 232448, "exceeds the 227 KB of shared memory a CTA can opt into");
};

// B_T: the GEMM also writes its B operand transposed to bt (store_b_transposed) -- each B tile once, from a stage that holds
// it for the product anyway.
template <bool A_MN, bool B_MN, class Epi, class AX = AXNone, bool B_T = false>
__global__ void __launch_bounds__(kThreads, 1)
umma_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmAlo, const __grid_constant__ CUtensorMap tmBlo, GemmShape gs,
                 GemmPtrs ptr, Epi epi, AX ax = AX{}, BTransposed bt = {}) {
  if (epi_gate_closed(epi, 0)) return;      // gated fallback pass: nothing to do (uniform over the grid)
  using L = SmemLayout;
  static_assert(!(A_MN && AX::kKind == 2), "the gathered A tile is K-major");
  constexpr bool kTmaA = !A_MN && AX::kKind == 0;     // K-major tiles TMA writes as wgmma reads them
  constexpr bool kTmaB = !B_MN;
  static_assert(!B_T || (kTmaA && kTmaB), "the B tile is copied out of all-K-major TMA stages");
  constexpr uint32_t kTxBytes = (kTmaA ? L::kABytes : 0) + (kTmaB ? L::kBBytes : 0);
  constexpr uint32_t kMnTxBytes = (A_MN ? L::kABytes : 0) + (B_MN ? L::kBBytes : 0);    // MN-major tiles, transposed after landing
  // How many steps the producer's TMA loads run ahead of the step it completes (transposes and publishes).  The
  // consumers free step i-1's stage only after issuing step i, so the producer must have published step i-STAGES+1
  // before it waits for the stage of step i: at most STAGES-2 steps ahead.
  constexpr int kLag = kMnTxBytes ? STAGES - 2 : 0;
  static_assert(kLag <= STAGES - 2, "the producer would wait for a stage only a step it has not published can free");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarOffset);     // the stage is ready for the MMA
  uint64_t* empty_bar = full_bar + STAGES;                                     // the MMA has read the stage
  uint64_t* landed_bar = empty_bar + STAGES;                                   // the MN-major boxes have landed
  uint64_t* epi_full = landed_bar + STAGES;                                    // the staging blocks hold a tile
  uint64_t* epi_empty = epi_full + 1;                                          // the epilogue is done with them

  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_items = gs.m_tiles * gs.n_tiles * gs.splits;
  const int total_kblocks = (gs.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    // B_T: producer warp 0 alone publishes a stage, and warps 1-3 release it like three more consumer warps
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], B_T ? 32 : 128);
      mbar_init(&empty_bar[s], B_T ? 8 + 3 : 8);
      mbar_init(&landed_bar[s], 1);
    }
    mbar_init(epi_full, 256);
    mbar_init(epi_empty, 128);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  auto decode = [&](int item, int& mt, int& nt, int& sp) {
    if (gs.n_fastest) {
      nt = item % gs.n_tiles;
      const int r = item / gs.n_tiles;
      mt = r % gs.m_tiles;
      sp = r / gs.m_tiles;
    } else {          // m fastest so CTAs running together share B tiles in L2
      mt = item % gs.m_tiles;
      const int r = item / gs.m_tiles;
      nt = r % gs.n_tiles;
      sp = r / gs.n_tiles;
    }
  };

  if (wg == 0) {
    // ===================== producer warpgroup =====================
    if constexpr (epi_move_regs<Epi>(0)) wg_regs_dec<kRegsProducer>();
    const int t = threadIdx.x;
    // The step sequence the consumers run: work items; per item, 3xTF32's three passes -- the two small cross terms
    // (A_lo.B_hi, A_hi.B_lo) over the whole K range first, then A_hi.B_hi (while only the 2^-11-sized cross terms have
    // been accumulated, the rounding of the fp32 accumulator costs nothing that matters, so the accumulation error is
    // that of ONE pass over K instead of three); per pass, the K blocks.  Cursors walk it: `ld` issues a step's loads,
    // `tr` completes the step kLag steps behind (all-K-major: one cursor does both).
    struct Cursor {
      int item, mt, nt, kb, kb0, kb1, pass;      // pass 0: A_lo.B_hi, 1: A_hi.B_lo, 2: A_hi.B_hi
      int stage;
      uint32_t phase;
    };
    auto seek = [&](Cursor& c) {                 // the first step of work item c.item or of the next one that has a step
      for (; c.item < total_items; c.item += gridDim.x) {
        int sp;
        decode(c.item, c.mt, c.nt, sp);
        c.kb = c.kb0 = sp * gs.kblocks_per_split;
        c.kb1 = min(total_kblocks, c.kb0 + gs.kblocks_per_split);
        c.pass = gs.terms == 3 ? 0 : 2;
        if (c.kb0 < c.kb1) return;
      }
    };
    auto next = [&](Cursor& c) {
      if (++c.stage == STAGES) { c.stage = 0; c.phase ^= 1; }
      if (++c.kb < c.kb1) return;
      if (c.pass < 2) { ++c.pass; c.kb = c.kb0; return; }
      c.item += gridDim.x;
      seek(c);
    };
    // issue: wait for the stage to be free; K-major TMA on full_bar, MN-major boxes on landed_bar; the loaders that
    // compute their A tile (gather, K-major softmax gradient) write it now
    auto issue = [&](const Cursor& c) {
      mbar_wait(&empty_bar[c.stage], c.phase ^ 1);
      uint8_t* sa = smem + c.stage * L::kStageBytes;
      uint8_t* sb = sa + L::kABytes;
      const int k0 = c.kb * BK;
      const bool a_lo = c.pass == 0, b_lo = c.pass == 1;
      if (t == 0) {
        if (kTxBytes) {
          mbar_expect_tx(&full_bar[c.stage], kTxBytes);
          if (kTmaA) tma_load_2d(sa, a_lo ? &tmAlo : &tmA, &full_bar[c.stage], k0, c.mt * BM);
          if (kTmaB) tma_load_2d(sb, b_lo ? &tmBlo : &tmB, &full_bar[c.stage], k0, c.nt * BN);
        }
        if (kMnTxBytes) {
          mbar_arrive_expect_tx(&landed_bar[c.stage], kMnTxBytes);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            if (A_MN) tma_load_2d(sa + q * 4096, a_lo ? &tmAlo : &tmA, &landed_bar[c.stage], c.mt * BM + 32 * q, k0);
            if (B_MN) tma_load_2d(sb + q * 4096, b_lo ? &tmBlo : &tmB, &landed_bar[c.stage], c.nt * BN + 32 * q, k0);
          }
        }
      }
      if constexpr (AX::kKind == 2) load_tile_gather(sa, ax, c.mt * BM, gs.M, c.kb, ax.Xout != nullptr && c.nt == 0, t);
      else if constexpr (!A_MN && !kTmaA) load_tile_k(sa, ptr.a, ptr.lda, c.mt * BM, gs.M, k0, gs.K, t, ax);
    };
    // complete: transpose the MN-major tiles in place (warp w: box w of each), then publish the stage
    auto complete = [&](const Cursor& c) {
      uint8_t* sa = smem + c.stage * L::kStageBytes;
      uint8_t* sb = sa + L::kABytes;
      if constexpr (kMnTxBytes != 0) {
        if constexpr (A_MN && AX::kKind == 1) {
          // S^T: tile K is examples.  Lane l fetches example k0 + l's (c, target) before the wait; element (x, k)
          // takes example k's from lane k.
          const int k0 = c.kb * BK, x = c.mt * BM + 32 * warp + lane;
          float ce = 0.f;
          int te = -1;
          if (k0 + lane < gs.K) ax.example(k0 + lane, ce, te);
          mbar_wait(&landed_bar[c.stage], c.phase);
          transpose_box(sa + warp * 4096, lane, [&](float s, int k) {
            const float ck = __shfl_sync(0xffffffffu, ce, k);
            const int tk = __shfl_sync(0xffffffffu, te, k);
            return (x < gs.M && k0 + k < gs.K) ? ax.p(s, x, ck, tk) : 0.f;
          });
        } else {
          mbar_wait(&landed_bar[c.stage], c.phase);
          if constexpr (A_MN) transpose_box(sa + warp * 4096, lane, [](float s, int) { return s; });
        }
        if constexpr (B_MN) transpose_box(sb + warp * 4096, lane, [](float s, int) { return s; });
      }
      if constexpr (!kTmaA || !kTmaB) fence_proxy_async_smem();     // generic-proxy stores -> visible to wgmma
      mbar_arrive(&full_bar[c.stage]);
    };
    Cursor ld{static_cast<int>(blockIdx.x), 0, 0, 0, 0, 0, 0, 0, 0u};
    seek(ld);
    if constexpr (B_T) {
      if (warp == 0) {          // the loads, never held up by the copy
        for (; ld.item < total_items; next(ld)) { issue(ld); complete(ld); }
      } else {
        // warps 1-3 walk the same steps: wait for the stage, copy its B tile out if this m-tile is the one that copies it
        // (3xTF32: B_lo of pass 1 to bt.lo, B_hi of pass 2 to bt.hi; pass 0 reads B_hi too), then release it -- in every
        // step, so that empty_bar's count holds whichever item a stage belongs to.  K block kb of n-tile nt is copied by
        // m-tile (nt + kb) % m_tiles: every work item, and so every CTA, copies its share of the blocks.  (Copying all of
        // them in m-tile 0 loaded the copy onto the quarter of the CTAs that run m-tile 0 items, and cost the logits GEMM
        // of the java14m step as much time as the separate pass it replaced.)
        for (; ld.item < total_items; next(ld)) {
          mbar_wait(&full_bar[ld.stage], ld.phase);
          if (ld.pass > 0 && (ld.nt + ld.kb) % gs.m_tiles == ld.mt)
            store_b_transposed(smem + ld.stage * L::kStageBytes + L::kABytes, ld.pass == 2 ? bt.hi : bt.lo, bt.ld, ld.nt * BN,
                               gs.N, ld.kb * BK, gs.K, warp - 1, lane);
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[ld.stage]);
        }
      }
    } else if constexpr (kLag == 0) {
      // all-K-major: one cursor (the lagging loop below, run with kLag = 0, was 10-19% slower on these GEMMs on an H100)
      for (; ld.item < total_items; next(ld)) { issue(ld); complete(ld); }
    } else {
      Cursor tr = ld;
      for (int ahead = 0; tr.item < total_items;) {      // ahead: steps issued and not yet completed
        const bool more = ld.item < total_items;
        if (more) { issue(ld); next(ld); ++ahead; }
        if (ahead > kLag || !more) { complete(tr); next(tr); --ahead; }
      }
    }
  } else if (wg <= 2) {
    // ===================== consumer warpgroups: rows 64 (wg - 1) .. of the tile =====================
    const int cw = wg - 1, wl = warp & 3;
    const int g = lane >> 2;      // this thread's rows of the accumulator: 16 wl + g (+ 8); columns 8 j + 2 (lane % 4) (+ 1)
    // staging: 8 blocks of 32 x 32 fp32 (row half, column quarter), 1024-byte aligned
    const uint32_t stg_row = smem_u32(smem + L::kEpiOffset + cw * L::kEpiBytes) + (wl >> 1) * 4096 + (16 * (wl & 1) + g) * 128 +
                             ((g ^ ((lane >> 1) & 1)) << 4) + 8 * (lane & 1);
    int stage = 0;
    uint32_t phase = 0, epi_phase = 0;
    float acc[64];
    for (int item = blockIdx.x; item < total_items; item += gridDim.x, epi_phase ^= 1) {
      int mt, nt, sp;
      decode(item, mt, nt, sp);
      const int kb0 = sp * gs.kblocks_per_split;
      const int kb1 = min(total_kblocks, kb0 + gs.kblocks_per_split);
      const int n_steps = (kb1 - kb0) * gs.terms;          // 3xTF32: three passes over the K range (see the producer)
      int prev = 0;
      for (int it = 0; it < n_steps; ++it) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * L::kStageBytes) + cw * 64 * 128;
        const uint32_t sb = smem_u32(smem + stage * L::kStageBytes + L::kABytes);
        wg_fence();
#pragma unroll
        for (int k = 0; k < BK / WG_K; ++k)
          wgmma_tf32(acc, gmma_desc(sa + k * WG_K * 4), gmma_desc(sb + k * WG_K * 4), (it > 0 || k > 0) ? 1u : 0u);
        wg_commit();
        wg_wait<1>();                                       // the previous stage's products have retired: release it
        if (it > 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wg_wait<0>();
      if (n_steps > 0 && lane == 0) mbar_arrive(&empty_bar[prev]);

      // Hand the tile to the epilogue warpgroup and go on to the next one.  The accumulator goes through shared
      // memory (8 XOR-swizzled 32 x 32 blocks per consumer: block (row half, column quarter)) so that an epilogue
      // thread then holds one row's 32 consecutive columns, the layout the functors' row-wise math and
      // store_chunk's coalesced stores work on.  The epilogue of this tile runs next to the MMAs of the next
      // one, which is only sound because no GEMM reads in its main loop what its epilogue writes: dY reads S and
      // v^T and updates (theta, m, v) of the target table, logits reads Ytab (or its tf32 split) and writes the
      // slab and the partials, and the other GEMMs write outputs that are none of their operands.
      // Element (row r, column cc) goes to block (r / 32, cc / 32), row r % 32, 16-byte chunk (cc % 32 / 4) ^ (r % 8).
      // For this thread's rows 16 wl + lane / 4 (+ 8 i) and columns 8 j + 2 (lane % 4) that is byte
      // (stg_row ^ ((j % 4) << 5)) + 8192 (j / 4) + 1024 i: written so, the 32 stores need four addresses, not 32
      // loop-invariant ones.
      mbar_wait(epi_empty, epi_phase ^ 1);                  // the epilogue is done with the previous tile's blocks
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
        for (int i = 0; i < 2; ++i)
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"((stg_row ^ ((j & 3) << 5)) + 8192 * (j >> 2) + 1024 * i),
                       "f"(acc[4 * j + 2 * i]), "f"(acc[4 * j + 2 * i + 1]) : "memory");
      }
      mbar_arrive(epi_full);
    }
  } else {
    // ===================== epilogue warpgroup: warp w drains rows 32w .. 32w+31 of the tile =====================
    // i.e. row half w & 1 of consumer w >> 1, all four column quarters.  The (max, sum) partial of slot 2 nt + p
    // takes column quarters p and p + 2, in that order.
    if constexpr (epi_move_regs<Epi>(0)) wg_regs_inc<kRegsEpilogue>();
    const int w = warp & 3;
    float* stg = reinterpret_cast<float*>(smem + L::kEpiOffset + (w >> 1) * L::kEpiBytes);
    auto prefetch_item = [&](int it) {            // read-modify-write epilogues: warm L2 with the tile's destination lines
      if (it >= total_items) return;
      int mt2, nt2, sp2;
      decode(it, mt2, nt2, sp2);
      epi_prefetch_tile(epi, mt2 * BM + 32 * w + lane, nt2 * BN, BN, gs.M, gs.N, 0);
    };
    prefetch_item(blockIdx.x);
    uint32_t epi_phase = 0;
    for (int item = blockIdx.x; item < total_items; item += gridDim.x, epi_phase ^= 1) {
      int mt, nt, sp;
      decode(item, mt, nt, sp);
      prefetch_item(item + gridDim.x);
      mbar_wait<true>(epi_full, epi_phase);
      const int m_base = mt * BM + 32 * w, m = m_base + lane;
      float* cbase = epi.out(sp);
#pragma unroll 1
      for (int p = 0; p < 2; ++p) {
        typename Epi::State est;
        epi.begin(est);
#pragma unroll 1
        for (int q = p; q < 4; q += 2) {
          float* blk = stg + ((w & 1) | (q << 1)) * 1024;
          uint32_t r[32];
#pragma unroll
          for (int c4 = 0; c4 < 8; ++c4) {
            const float4 x = *reinterpret_cast<const float4*>(blk + lane * 32 + ((c4 ^ (lane & 7)) << 2));
            r[4 * c4] = __float_as_uint(x.x); r[4 * c4 + 1] = __float_as_uint(x.y);
            r[4 * c4 + 2] = __float_as_uint(x.z); r[4 * c4 + 3] = __float_as_uint(x.w);
          }
          __syncwarp();
          const int n = nt * BN + 32 * q;
          if (n < gs.N) {
            if (m < gs.M) epi.observe(m, n, r, gs.N - n, est);
            if (epi_stores<Epi>(0)) store_chunk(epi, est, r, blk, lane, m_base, n, gs.M, gs.N, cbase, epi.ldc);
          }
        }
        epi.end(m, 2 * nt + p, sp, m < gs.M, est);
      }
      mbar_arrive(epi_empty);
    }
  }
}

// ---- host side ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && p)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D fp32 tensor map over a row-major [rows, cols] matrix with row pitch ld (floats); box = {32 cols, box_rows},
// SWIZZLE_128B.  Encoded maps are kept in a small per-thread cache: a training step issues the same dozen
// (buffer, shape) combinations every time, so after the first step no launch calls into the driver for a descriptor.
struct TensorMapKey {
  const float* base;
  uint64_t rows, cols, ld;
  uint32_t box_rows;
  bool operator==(const TensorMapKey& o) const {
    return base == o.base && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows;
  }
};
struct TensorMapCache {
  static constexpr int kCap = 96;
  TensorMapKey key[kCap];
  CUtensorMap map[kCap];
  int n = 0, next = 0;
};
inline bool make_tensor_map(CUtensorMap* map, const float* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  static thread_local TensorMapCache cache;
  const TensorMapKey k{base, rows, cols, ld, box_rows};
  for (int i = 0; i < cache.n; ++i)
    if (cache.key[i] == k) { *map = cache.map[i]; return true; }
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return false;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * sizeof(float)};
  cuuint32_t box[2] = {32, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return false;
  const int slot = (cache.n < TensorMapCache::kCap) ? cache.n++ : (cache.next++ % TensorMapCache::kCap);
  cache.key[slot] = k;
  cache.map[slot] = *map;
  return true;
}

// Operand description: `major_mn == false`: element (x, k) at base[x*ld + k] (K contiguous);
//                      `major_mn == true` : element (x, k) at base[k*ld + x] (M / N contiguous).
// 3xTF32 (C2V_MATH_3XTF32): `base` holds the tf32-rounded high parts and `lo` (same layout) the tf32-rounded
// residuals x - hi; both operands of a product must carry one, or neither.
struct Operand {
  const float* base;
  size_t ld;
  bool major_mn;
  const float* lo = nullptr;
};

// The tensor map of an operand with X rows (M or N) and depth K: K-major, boxes of 32 k x 128 rows, as wgmma reads
// them; MN-major, boxes of 32 x x 32 k-rows, four per stage, that the producer transposes.
inline bool operand_map(CUtensorMap* map, const float* base, bool major_mn, int X, int K, size_t ld) {
  return major_mn ? make_tensor_map(map, base, (uint64_t)K, (uint64_t)X, ld, BK) : make_tensor_map(map, base, (uint64_t)X, (uint64_t)K, ld, BM);
}

inline GemmShape make_shape(int M, int N, int K, int splits, int terms) {
  GemmShape gs;
  gs.M = M; gs.N = N; gs.K = K;
  gs.terms = terms;
  gs.m_tiles = (M + BM - 1) / BM;
  gs.n_tiles = (N + BN - 1) / BN;
  const int total_kblocks = (K + BK - 1) / BK;
  if (splits < 1) splits = 1;
  if (splits > total_kblocks) splits = total_kblocks;
  gs.kblocks_per_split = (total_kblocks + splits - 1) / splits;
  gs.splits = (total_kblocks + gs.kblocks_per_split - 1) / gs.kblocks_per_split;
  // few, wide n-tiles under many m-tiles: walk n fastest so the (large) A tile is fetched from HBM once
  gs.n_fastest = (gs.n_tiles < gs.m_tiles) ? 1 : 0;
  return gs;
}

template <bool A_MN, bool B_MN, class Epi, class AX, bool B_T = false>
inline cudaError_t launch_kernel(cudaStream_t st, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmAlo,
                                 const CUtensorMap& tmBlo, const GemmShape& gs, const GemmPtrs& ptr, const Epi& epi, int num_sms,
                                 const AX& ax, const BTransposed& bt = {}) {
  auto kern = umma_gemm_kernel<A_MN, B_MN, Epi, AX, B_T>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemLayout::kTotal);
  if (e != cudaSuccess) return e;
  int grid = gs.m_tiles * gs.n_tiles * gs.splits;
  if (grid > num_sms) grid = num_sms;
  kern<<<grid, kThreads, SmemLayout::kTotal, st>>>(tmA, tmB, tmAlo, tmBlo, gs, ptr, epi, ax, bt);
  return cudaGetLastError();
}

// B_T: B^T [K, bt.ld] is written to bt as well (umma_gemm_kernel); bt.ld >= N, both 16-byte aligned with a pitch of a
// multiple of 4 floats, K % 4 == 0.
template <bool A_MN, bool B_MN, class Epi, class AX = AXNone, bool B_T = false>
inline cudaError_t launch_cfg(cudaStream_t st, int M, int N, int K, int splits, const Operand& A, const Operand& B, const Epi& epi,
                              int num_sms, const AX& ax = AX{}, const BTransposed& bt = {}) {
  CUtensorMap tmA{}, tmB{}, tmAlo{}, tmBlo{};
  const bool three = A.lo != nullptr && B.lo != nullptr;
  if ((A.lo != nullptr) != (B.lo != nullptr)) return cudaErrorInvalidValue;
  if (AX::kKind != 0 && three) return cudaErrorInvalidValue;      // the transforms rewrite a single fp32 tile
  if (B_T && (!bt.hi || (three && !bt.lo) || bt.ld < (size_t)N || bt.ld % 4 || K % 4 ||
              ((reinterpret_cast<uintptr_t>(bt.hi) | reinterpret_cast<uintptr_t>(bt.lo)) % 16)))
    return cudaErrorInvalidValue;
  if (A_MN || AX::kKind == 0) {
    if (!operand_map(&tmA, A.base, A_MN, M, K, A.ld)) return cudaErrorInvalidValue;
    if (three && !operand_map(&tmAlo, A.lo, A_MN, M, K, A.ld)) return cudaErrorInvalidValue;
  }
  if (!operand_map(&tmB, B.base, B_MN, N, K, B.ld)) return cudaErrorInvalidValue;
  if (three && !operand_map(&tmBlo, B.lo, B_MN, N, K, B.ld)) return cudaErrorInvalidValue;
  const GemmPtrs ptr{A.base, A.ld};
  return launch_kernel<A_MN, B_MN, Epi, AX, B_T>(st, tmA, tmB, tmAlo, tmBlo, make_shape(M, N, K, splits, three ? 3 : 1), ptr, epi,
                                                 num_sms, ax, bt);
}

// number of split-K slices launch_cfg will actually produce
inline int effective_splits(int K, int splits) {
  const int total_kblocks = (K + BK - 1) / BK;
  if (splits < 1) splits = 1;
  if (splits > total_kblocks) splits = total_kblocks;
  const int per = (total_kblocks + splits - 1) / splits;
  return (total_kblocks + per - 1) / per;
}

// (max, sum exp) partial slots per logits row: one per (row, tile, parity of the tile's 32-column quarter)
inline int lse_slots(int n) { return 2 * ((n + BN - 1) / BN); }

// Runtime dispatch over operand majors.
template <class Epi>
inline cudaError_t launch(cudaStream_t st, int M, int N, int K, int splits, const Operand& A, const Operand& B, const Epi& epi,
                          int num_sms) {
  if (!A.major_mn && !B.major_mn) return launch_cfg<false, false, Epi>(st, M, N, K, splits, A, B, epi, num_sms);
  if (!A.major_mn && B.major_mn) return launch_cfg<false, true, Epi>(st, M, N, K, splits, A, B, epi, num_sms);
  if (A.major_mn && !B.major_mn) return launch_cfg<true, false, Epi>(st, M, N, K, splits, A, B, epi, num_sms);
  return launch_cfg<true, true, Epi>(st, M, N, K, splits, A, B, epi, num_sms);
}

// Fused context forward:  H[M, N] = epi( dropout(gather(cs))[M, K = 3d] . W[K, N] )  (tensorflow_model.py:238-252)
// in one kernel -- the producer warpgroup gathers the embedding rows straight into the swizzled A stage, so the
// gathered context matrix X' is never read back from HBM.  W row-major [K, N] (N contiguous).  Xout: nullptr or
// [M, K] (written once when a backward pass needs X').  Precondition (checked by the caller): d % 32 == 0.
template <class Epi>
inline cudaError_t launch_ctx_fused(cudaStream_t st, int M, int N, const float* W, size_t ldw, const ContextSource& cs,
                                    const Dropout& dp, float* Xout, const Epi& epi, int num_sms) {
  const int K = 3 * cs.d;
  GemmShape gs = make_shape(M, N, K, 1, 1);
  gs.n_fastest = 1;          // the CTAs that run together share gathered rows through L2
  const CUtensorMap none{};
  CUtensorMap tmW{};
  if (!operand_map(&tmW, W, true, N, K, ldw)) return cudaErrorInvalidValue;
  return launch_kernel<false, true, Epi, AXGather>(st, none, tmW, none, none, gs, GemmPtrs{nullptr, 0}, epi, num_sms, AXGather{cs, dp, Xout});
}

// TMA constraints on an operand of either major: 16-byte aligned base, row pitch a multiple of 16 bytes.
inline bool operand_ok(const Operand& o) {
  return (reinterpret_cast<uintptr_t>(o.base) % 16 == 0) && (o.ld % 4 == 0);
}

}  // namespace umma
}  // namespace c2v
