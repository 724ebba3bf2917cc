// Nearest-neighbour search over the rows of a float32 table (include/c2v_b200.h "Nearest neighbours", DESIGN.md §6h):
// gensim's KeyedVectors.most_similar on the embedding tables, and the nearest methods of a corpus by code vector.
//   bind    : norm_i = ||T_i|| in double; inv_norm_i = 1 / norm_i as float (inf for a zero row, whose scores are then
//             0 * inf = NaN and never enter a list).  The GEMM reads the table through a copy with a 16-byte row pitch
//             (zero columns up to dim rounded to 4) when the caller's table has none, and as its tf32 split in 3xTF32.
//   queries : one block per query; sum_w weight_w T_w / norm_w in double, scaled to unit length (a zero sum stays zero).
//   search  : queries go in blocks whose candidate lists (or slab) fit kBlockBytes.  Per block:
//             tensor cores (tf32, 3xTF32; k + excluded <= kTopkEpiMax): the wgmma GEMM Q . T^T with T as the K-major B,
//               whose epilogue (EpiKnnT) scales column j by inv_norm_j and keeps each (row, slot)'s best candidates, then
//               the engine's topk_merge_kernel merges a row's slots;
//             slab (fp32, or more candidates): the SIMT GEMM writes the scaled scores [rows, N], the engine's topk
//               kernels pick from each row;
//             then exclude_kernel drops each query's excluded ids and keeps the first k of the rest.
#include <cuda_runtime.h>
#include <limits.h>
#include <math.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/c2v_b200.h"
#include "common.cuh"
#include "sgemm.cuh"
#include "umma_gemm.cuh"

namespace c2v {
void set_global_error(const std::string& msg);     // engine.cu: the message c2v_last_error(NULL) returns
cudaError_t knn_topk_merge(const int32_t* idx, const float* val, int L, int k, int rows, int32_t* idx_out, float* val_out,
                           cudaStream_t st);
cudaError_t knn_topk_slab(const float* S, size_t ldS, int N, int k, int rows, int32_t* idx_out, float* val_out, cudaStream_t st);

namespace umma {
// EpiTopkT's candidate lists over scores instead of dot products: column j's accumulator is multiplied by inv_norm[j]
// before the screen and the insert.  A NaN score (zero or NaN row) never passes the strict comparison.
template <bool PRECISE>
struct EpiKnnT : EpiTopkT<PRECISE, false> {
  using Base = EpiTopkT<PRECISE, false>;
  const float* inv_norm;    // [N]
  __device__ __forceinline__ void observe(int m, int n, const uint32_t (&r)[32], int nvalid, typename Base::State& st) const {
    uint32_t s[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) s[j] = __float_as_uint(j < nvalid ? __uint_as_float(r[j]) * __ldg(inv_norm + n + j) : 0.f);
    Base::observe(m, n, s, nvalid, st);
  }
};
}  // namespace umma
}  // namespace c2v

namespace {
using namespace c2v;

// Candidate lists or the score slab of one query block take at most this much device memory.
constexpr size_t kBlockBytes = size_t(512) << 20;
constexpr int64_t kMaxBlockRows = 1 << 16;     // and hold at most this many queries (their fp32 copy, the merged lists)
constexpr int kSlabMax = 64;           // topk_iter_kernel's largest k

// rows of x [rows, dim] (pitch ld) -> out [rows, ldp] with zero columns dim .. ldp-1; lo != nullptr: the tf32 split
__global__ void __launch_bounds__(256)
pad_split_kernel(const float* __restrict__ x, int64_t rows, int dim, int64_t ld, float* __restrict__ out,
                 float* __restrict__ lo, int ldp) {
  const int64_t n = rows * ldp;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
    const int64_t r = i / ldp;
    const int c = (int)(i - r * ldp);
    const float v = c < dim ? x[r * ld + c] : 0.f;
    if (lo) {
      float h, l;
      split_tf32(v, h, l);
      out[i] = h;
      lo[i] = l;
    } else {
      out[i] = v;
    }
  }
}

// one warp per row: norm in double, and the float reciprocal the scores use
__global__ void __launch_bounds__(256)
norm_kernel(const float* __restrict__ x, int64_t rows, int dim, int64_t ld, double* __restrict__ norm,
            float* __restrict__ inv_norm) {
  const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  double s = 0.0;
  for (int c = lane; c < dim; c += 32) {
    const double v = x[r * ld + c];
    s += v * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    const double nr = sqrt(s);
    norm[r] = nr;
    inv_norm[r] = (float)(1.0 / nr);
  }
}

__device__ __forceinline__ double block_sum_d(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
  return t;
}

// gensim's query: sum of weight_w T_w / norm_w over words [off[q], off[q + 1]), then unitvec (a zero sum stays zero)
__global__ void __launch_bounds__(128)
query_kernel(const float* __restrict__ T, int64_t ld, int dim, const double* __restrict__ norm, const int32_t* __restrict__ ids,
             const float* __restrict__ w, const int64_t* __restrict__ off, float* __restrict__ q) {
  __shared__ double red[4];
  const int64_t a = off[blockIdx.x], b = off[blockIdx.x + 1];
  auto at = [&](int c) {
    double s = 0.0;
    for (int64_t j = a; j < b; ++j) s += (double)w[j] * (double)T[(int64_t)ids[j] * ld + c] / norm[ids[j]];
    return s;
  };
  double ss = 0.0;
  for (int c = threadIdx.x; c < dim; c += 128) {
    const double s = at(c);
    ss += s * s;
  }
  ss = block_sum_d(ss, red);
  const double scale = ss > 0.0 ? 1.0 / sqrt(ss) : 1.0;
  for (int c = threadIdx.x; c < dim; c += 128) q[(int64_t)blockIdx.x * dim + c] = (float)(at(c) * scale);
}

// C[m, n] = acc * inv_norm[n]: the slab route's scores
struct ScaledStore {
  float* C;
  size_t ldc;
  const float* inv_norm;
  __device__ __forceinline__ void operator()(int m, int n, const float4& v, int nvalid) const {
    float4 s;
    s.x = v.x * inv_norm[n];
    s.y = nvalid > 1 ? v.y * inv_norm[n + 1] : 0.f;
    s.z = nvalid > 2 ? v.z * inv_norm[n + 2] : 0.f;
    s.w = nvalid > 3 ? v.w * inv_norm[n + 3] : 0.f;
    simt::st4_guard(C + (size_t)m * ldc + n, s, nvalid);
  }
};

// query r of the block: its kk ranked candidates minus the ids exclude[xoff[r0 + r], xoff[r0 + r + 1]) (every copy of an
// excluded id goes), the first k of the rest, padded with (-inf, INT_MAX)
__global__ void __launch_bounds__(128)
exclude_kernel(const int32_t* __restrict__ midx, const float* __restrict__ mval, int rows, int kk, int k,
               const int32_t* __restrict__ ex, const int64_t* __restrict__ xoff, int64_t r0, int32_t* __restrict__ idx,
               float* __restrict__ val) {
  const int r = blockIdx.x * 128 + threadIdx.x;
  if (r >= rows) return;
  const int64_t a = xoff ? xoff[r0 + r] : 0, b = xoff ? xoff[r0 + r + 1] : 0;
  int o = 0;
  for (int j = 0; j < kk && o < k; ++j) {
    const int32_t id = midx[(size_t)r * kk + j];
    bool drop = false;
    for (int64_t e = a; e < b && !drop; ++e) drop = ex[e] == id && id != INT_MAX;
    if (drop) continue;
    idx[(size_t)r * k + o] = id;
    val[(size_t)r * k + o] = mval[(size_t)r * kk + j];
    ++o;
  }
  for (; o < k; ++o) {
    idx[(size_t)r * k + o] = INT_MAX;
    val[(size_t)r * k + o] = -INFINITY;
  }
}

struct Buf {
  void* p = nullptr;
  size_t bytes = 0;
};

}  // namespace

struct c2v_knn {
  int device = 0;
  int num_sms = 0;
  // the bound table
  const float* table = nullptr;
  int64_t rows = 0, ld = 0;
  int dim = 0, ldp = 0, math = C2V_MATH_3XTF32;
  const float* plain = nullptr;    // the table in fp32 with a 16-byte row pitch: the caller's, or t_pad (pitch ldp)
  int64_t plain_ld = 0;
  Buf norm, inv_norm, t_pad, t_hi, t_lo;
  // per query block
  Buf q_hi, q_lo, cand, slab, merged;
  size_t held = 0, peak = 0;
  bool profile = false;
  std::vector<cudaEvent_t> events;          // (start, after the GEMM, after the selection) per profiled block
  double gemm_ms = 0.0, select_ms = 0.0;
};

namespace {

int kfail(int code, const std::string& msg) {
  c2v::set_global_error(msg);
  return code;
}
int kcuda(const char* fn, cudaError_t e) { return kfail(C2V_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(e)); }
#define KCHECK(fn, expr)                        \
  do {                                          \
    cudaError_t _c = (expr);                    \
    if (_c != cudaSuccess) return kcuda(fn, _c); \
  } while (0)

// b holds at least `bytes` (contents not kept)
cudaError_t reserve(c2v_knn* h, Buf& b, size_t bytes) {
  if (b.bytes >= bytes) return cudaSuccess;
  if (b.p) {
    cudaFree(b.p);
    h->held -= b.bytes;
    b.p = nullptr;
    b.bytes = 0;
  }
  cudaError_t e = cudaMalloc(&b.p, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return e;
  }
  b.bytes = bytes;
  h->held += bytes;
  if (h->held > h->peak) h->peak = h->held;
  return cudaSuccess;
}

void release(c2v_knn* h, Buf& b) {
  if (b.p) cudaFree(b.p);
  h->held -= b.bytes;
  b = Buf{};
}

unsigned grid_for(int64_t n, int num_sms) {
  int64_t g = (n + 255) / 256;
  if (g > (int64_t)num_sms * 16) g = (int64_t)num_sms * 16;
  return (unsigned)(g < 1 ? 1 : g);
}

template <bool X3>
cudaError_t launch_epilogue_gemm(c2v_knn* h, cudaStream_t st, int nb, int kk, float* cval, int32_t* cidx) {
  umma::Operand A{static_cast<float*>(h->q_hi.p), (size_t)h->ldp, false, X3 ? static_cast<float*>(h->q_lo.p) : nullptr};
  umma::Operand B = X3 ? umma::Operand{static_cast<float*>(h->t_hi.p), (size_t)h->ldp, false, static_cast<float*>(h->t_lo.p)}
                       : umma::Operand{h->plain, (size_t)h->plain_ld, false};
  const int N = (int)h->rows;
  const umma::EpiStoreLseT<X3> none{nullptr, 0, nullptr, umma::lse_slots(N)};
  const umma::EpiKnnT<X3> epi{{none, cval, cidx, kk, 0}, static_cast<const float*>(h->inv_norm.p)};
  return umma::launch_cfg<false, false, umma::EpiKnnT<X3>>(st, nb, N, h->ldp, 1, A, B, epi, h->num_sms);
}

}  // namespace

extern "C" {

int c2v_knn_create(int device, c2v_knn** out) {
  if (!out) return kfail(C2V_ERR_INVALID, "c2v_knn_create: NULL out");
  *out = nullptr;
  KCHECK("c2v_knn_create", cudaSetDevice(device));
  cudaDeviceProp prop;
  KCHECK("c2v_knn_create", cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9) return kfail(C2V_ERR_UNSUPPORTED, "c2v_knn_create: the kernels are built for sm_90a (H100)");
  c2v_knn* h = new c2v_knn();
  h->device = device;
  h->num_sms = prop.multiProcessorCount;
  *out = h;
  return C2V_OK;
}

void c2v_knn_destroy(c2v_knn* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  for (Buf* b : {&h->norm, &h->inv_norm, &h->t_pad, &h->t_hi, &h->t_lo, &h->q_hi, &h->q_lo, &h->cand, &h->slab, &h->merged})
    if (b->p) cudaFree(b->p);
  for (cudaEvent_t ev : h->events) cudaEventDestroy(ev);
  delete h;
}

size_t c2v_knn_device_bytes(const c2v_knn* h) { return h ? h->peak : 0; }

int c2v_knn_bind_table(c2v_knn* h, const float* table, int64_t rows, int32_t dim, int64_t ld, int32_t math, void* stream) {
  const char* fn = "c2v_knn_bind_table";
  if (!h || !table) return kfail(C2V_ERR_INVALID, std::string(fn) + ": NULL handle or table");
  if (rows < 1 || rows >= INT_MAX || dim < 1 || ld < dim)
    return kfail(C2V_ERR_INVALID, std::string(fn) + ": need 1 <= rows < 2^31 and 1 <= dim <= ld");
  if (math < C2V_MATH_FP32 || math > C2V_MATH_3XTF32) return kfail(C2V_ERR_INVALID, std::string(fn) + ": math must be 0, 1 or 2");
  KCHECK(fn, cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  h->table = nullptr;
  const int ldp = (dim + 3) / 4 * 4;
  const bool aligned = dim % 4 == 0 && ld % 4 == 0 && reinterpret_cast<uintptr_t>(table) % 16 == 0;
  const bool x3 = math == C2V_MATH_3XTF32;
  KCHECK(fn, reserve(h, h->norm, (size_t)rows * 8));
  KCHECK(fn, reserve(h, h->inv_norm, (size_t)rows * 4));
  if (!aligned) KCHECK(fn, reserve(h, h->t_pad, (size_t)rows * ldp * 4));
  else release(h, h->t_pad);
  if (x3) {
    KCHECK(fn, reserve(h, h->t_hi, (size_t)rows * ldp * 4));
    KCHECK(fn, reserve(h, h->t_lo, (size_t)rows * ldp * 4));
  } else {
    release(h, h->t_hi);
    release(h, h->t_lo);
  }
  norm_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(table, rows, dim, ld, static_cast<double*>(h->norm.p),
                                                           static_cast<float*>(h->inv_norm.p));
  KCHECK(fn, cudaGetLastError());
  if (!aligned) {
    pad_split_kernel<<<grid_for(rows * ldp, h->num_sms), 256, 0, st>>>(table, rows, dim, ld, static_cast<float*>(h->t_pad.p),
                                                                        nullptr, ldp);
    KCHECK(fn, cudaGetLastError());
  }
  if (x3) {
    pad_split_kernel<<<grid_for(rows * ldp, h->num_sms), 256, 0, st>>>(table, rows, dim, ld, static_cast<float*>(h->t_hi.p),
                                                                        static_cast<float*>(h->t_lo.p), ldp);
    KCHECK(fn, cudaGetLastError());
  }
  h->table = table;
  h->rows = rows;
  h->dim = dim;
  h->ld = ld;
  h->ldp = ldp;
  h->math = math;
  h->plain = aligned ? table : static_cast<const float*>(h->t_pad.p);
  h->plain_ld = aligned ? ld : ldp;
  return C2V_OK;
}

int c2v_knn_queries(c2v_knn* h, const int32_t* word_ids, const float* weights, const int64_t* offsets, int32_t nq, float* q_out,
                    void* stream) {
  const char* fn = "c2v_knn_queries";
  if (!h || !h->table) return kfail(C2V_ERR_STATE, std::string(fn) + ": no table bound");
  if (nq < 0 || (nq > 0 && (!word_ids || !weights || !offsets || !q_out)))
    return kfail(C2V_ERR_INVALID, std::string(fn) + ": NULL argument or nq < 0");
  if (nq == 0) return C2V_OK;
  KCHECK(fn, cudaSetDevice(h->device));
  query_kernel<<<nq, 128, 0, static_cast<cudaStream_t>(stream)>>>(h->table, h->ld, h->dim, static_cast<const double*>(h->norm.p),
                                                                   word_ids, weights, offsets, q_out);
  KCHECK(fn, cudaGetLastError());
  return C2V_OK;
}

int c2v_knn_search(c2v_knn* h, const float* q, int32_t nq, int64_t ldq, int32_t k, const int32_t* exclude,
                   const int64_t* exclude_off, int32_t max_exclude, int32_t* idx, float* val, void* stream) {
  const char* fn = "c2v_knn_search";
  if (!h || !h->table) return kfail(C2V_ERR_STATE, std::string(fn) + ": no table bound");
  if (nq < 0 || k < 1 || max_exclude < 0 || ldq < h->dim || (nq > 0 && (!q || !idx || !val)) ||
      (max_exclude > 0 && (!exclude || !exclude_off)))
    return kfail(C2V_ERR_INVALID, std::string(fn) + ": need k >= 1, max_exclude >= 0, ldq >= dim and non-NULL buffers");
  const int kk = k + max_exclude;
  if (kk > kSlabMax)
    return kfail(C2V_ERR_UNSUPPORTED, std::string(fn) + ": k + max_exclude = " + std::to_string(kk) + " exceeds " +
                                          std::to_string(kSlabMax));
  if (nq == 0) return C2V_OK;
  KCHECK(fn, cudaSetDevice(h->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int N = (int)h->rows;
  const bool tc = h->math != C2V_MATH_FP32 && kk <= umma::kTopkEpiMax;
  const bool x3 = tc && h->math == C2V_MATH_3XTF32;      // the slab route reads the fp32 table and queries
  const int slots = umma::lse_slots(N);
  const size_t ldS = (size_t)(N + 3) / 4 * 4;
  const size_t per_query = tc ? (size_t)slots * kk * 8 : ldS * 4;
  int64_t nb = (int64_t)(kBlockBytes / per_query);
  if (nb >= umma::BM) nb -= nb % umma::BM;              // whole GEMM row tiles
  if (nb < 1) nb = 1;
  if (nb > kMaxBlockRows) nb = kMaxBlockRows;
  if (nb > nq) nb = nq;
  KCHECK(fn, reserve(h, h->q_hi, (size_t)nb * h->ldp * 4));
  if (x3) KCHECK(fn, reserve(h, h->q_lo, (size_t)nb * h->ldp * 4));
  KCHECK(fn, reserve(h, tc ? h->cand : h->slab, (size_t)nb * per_query));
  KCHECK(fn, reserve(h, h->merged, (size_t)nb * kk * 8));
  int32_t* midx = static_cast<int32_t*>(h->merged.p);
  float* mval = reinterpret_cast<float*>(midx + (size_t)nb * kk);
  for (int64_t r0 = 0; r0 < nq; r0 += nb) {
    const int rows = (int)(nq - r0 < nb ? nq - r0 : nb);
    cudaEvent_t ev[3] = {};
    if (h->profile) {
      for (int i = 0; i < 3; ++i) {
        KCHECK(fn, cudaEventCreate(&ev[i]));
        h->events.push_back(ev[i]);
      }
      KCHECK(fn, cudaEventRecord(ev[0], st));
    }
    pad_split_kernel<<<grid_for((int64_t)rows * h->ldp, h->num_sms), 256, 0, st>>>(
        q + r0 * ldq, rows, h->dim, ldq, static_cast<float*>(h->q_hi.p), x3 ? static_cast<float*>(h->q_lo.p) : nullptr, h->ldp);
    KCHECK(fn, cudaGetLastError());
    if (tc) {
      float* cval = static_cast<float*>(h->cand.p);
      int32_t* cidx = reinterpret_cast<int32_t*>(cval + (size_t)rows * slots * kk);
      KCHECK(fn, x3 ? launch_epilogue_gemm<true>(h, st, rows, kk, cval, cidx) : launch_epilogue_gemm<false>(h, st, rows, kk, cval, cidx));
      if (h->profile) KCHECK(fn, cudaEventRecord(ev[1], st));
      KCHECK(fn, knn_topk_merge(cidx, cval, slots, kk, rows, midx, mval, st));
    } else {
      float* S = static_cast<float*>(h->slab.p);
      const simt::RowsK al{static_cast<const float*>(h->q_hi.p), (size_t)h->ldp};
      const simt::RowsK bl{h->plain, (size_t)h->plain_ld};
      KCHECK(fn, simt::launch(st, rows, N, h->ldp, 1, al, bl, ScaledStore{S, ldS, static_cast<const float*>(h->inv_norm.p)}));
      if (h->profile) KCHECK(fn, cudaEventRecord(ev[1], st));
      KCHECK(fn, knn_topk_slab(S, ldS, N, kk, rows, midx, mval, st));
    }
    exclude_kernel<<<(rows + 127) / 128, 128, 0, st>>>(midx, mval, rows, kk, k, exclude, max_exclude ? exclude_off : nullptr, r0,
                                                       idx + r0 * k, val + r0 * k);
    KCHECK(fn, cudaGetLastError());
    if (h->profile) KCHECK(fn, cudaEventRecord(ev[2], st));
  }
  return C2V_OK;
}

int c2v_knn_profile(c2v_knn* h, int32_t on, double* gemm_ms, double* select_ms) {
  if (!h) return kfail(C2V_ERR_INVALID, "c2v_knn_profile: NULL handle");
  KCHECK("c2v_knn_profile", cudaSetDevice(h->device));
  for (size_t i = 0; i + 3 <= h->events.size(); i += 3) {
    float a = 0.f, b = 0.f;
    KCHECK("c2v_knn_profile", cudaEventSynchronize(h->events[i + 2]));
    KCHECK("c2v_knn_profile", cudaEventElapsedTime(&a, h->events[i], h->events[i + 1]));
    KCHECK("c2v_knn_profile", cudaEventElapsedTime(&b, h->events[i + 1], h->events[i + 2]));
    h->gemm_ms += a;
    h->select_ms += b;
  }
  for (cudaEvent_t ev : h->events) cudaEventDestroy(ev);
  h->events.clear();
  if (gemm_ms) *gemm_ms = h->gemm_ms;
  if (select_ms) *select_ms = h->select_ms;
  h->gemm_ms = h->select_ms = 0.0;
  h->profile = on != 0;
  return C2V_OK;
}

}  // extern "C"
