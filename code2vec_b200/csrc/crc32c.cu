// CRC-32C on the device (include/c2v_b200.h "CRC-32C of device memory", DESIGN.md §6k): the checksum every entry of a
// TensorFlow tensor bundle carries, computed where the tensor's bytes already are.
// CRC-32C: reflected polynomial 0x82F63B78, init and xorout 0xFFFFFFFF.  Everything below works on the raw (init 0, no
// xorout) CRC, which is linear over GF(2):
//   raw(A || B)        = raw(A) * x^(8|B|) ^ raw(B)                        (products mod P, in the reflected order)
//   crc(M)             = raw(M) ^ 0xFFFFFFFF * x^(8|M|) ^ 0xFFFFFFFF
//   crc(A || B)        = crc(A) * x^(8|B|) ^ crc(B)                         (zlib's crc32_combine)
//   rows kernel    : one thread per 256-byte segment of a row: the raw CRC of its bytes by a byte table (32 copies in
//                    shared memory, copy c in bank c, so a warp's lookups never conflict), times x^(8 * the bytes after
//                    it in the row), XORed into the row's output word (zeroed first); segment 0 also XORs in the
//                    row-length constant above.  XOR is exact and order-free, so the result does not depend on timing.
//   combine kernel : a tree over 2048 leaves per block (8 per thread in sequence, then the warp, then the block), each
//                    level a product by the constant x^(8 * the right half's bytes); the sequence is padded at the
//                    front with zero leaves (a zero contributes nothing), and each block's result, times x^(8 * the
//                    bytes after the block), is XORed into *out.
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/c2v_b200.h"

namespace c2v {
void set_global_error(const std::string& msg);     // engine.cu: the message c2v_last_error(NULL) returns
}

namespace {

constexpr uint32_t kPoly = 0x82F63B78u;
constexpr uint32_t kOne = 0x80000000u;             // x^0 in the reflected order
constexpr int kThreads = 256;
constexpr int64_t kSeg = 256;                       // bytes per thread in the rows kernel
constexpr int kRun = 8;                             // leaves each thread folds in sequence in the combine kernel
constexpr int64_t kLeavesPerBlock = (int64_t)kThreads * kRun;

// a * b mod P (zlib's multmodp)
__host__ __device__ __forceinline__ uint32_t mulmodp(uint32_t a, uint32_t b) {
  uint32_t p = 0;
#pragma unroll 4
  for (int i = 0; i < 32; ++i) {
    if (a & (kOne >> i)) p ^= b;
    b = (b & 1u) ? (b >> 1) ^ kPoly : b >> 1;
  }
  return p;
}

struct PowTable {
  uint32_t v[64];                                   // v[j] = x^(8 * 2^j) mod P
};

constexpr PowTable make_pow_table() {
  PowTable t{};
  uint32_t x8 = kOne;
  for (int i = 0; i < 8; ++i) x8 = (x8 & 1u) ? (x8 >> 1) ^ kPoly : x8 >> 1;       // x^8
  t.v[0] = x8;
  for (int j = 1; j < 64; ++j) {
    uint32_t a = t.v[j - 1], b = t.v[j - 1], p = 0;
    for (int i = 0; i < 32; ++i) {
      if (a & (kOne >> i)) p ^= b;
      b = (b & 1u) ? (b >> 1) ^ kPoly : b >> 1;
    }
    t.v[j] = p;
  }
  return t;
}

constexpr PowTable kPowHost = make_pow_table();
__constant__ PowTable kPowDev = make_pow_table();

// x^(8 n) mod P from the table in `pw` (shared or host memory)
__host__ __device__ __forceinline__ uint32_t xpow8(uint64_t n, const uint32_t* pw) {
  uint32_t p = kOne;
  for (int j = 0; n; ++j, n >>= 1)
    if (n & 1u) p = mulmodp(pw[j], p);
  return p;
}

// the byte table, entry i of copy c at word i * 32 + c
__device__ void fill_table(uint32_t* table, uint32_t* pw) {
  for (int w = threadIdx.x; w < 256 * 32; w += blockDim.x) {
    uint32_t c = (uint32_t)w >> 5;
#pragma unroll
    for (int k = 0; k < 8; ++k) c = (c & 1u) ? (c >> 1) ^ kPoly : c >> 1;
    table[w] = c;
  }
  if (threadIdx.x < 64) pw[threadIdx.x] = kPowDev.v[threadIdx.x];
  __syncthreads();
}

__device__ __forceinline__ uint32_t crc_byte(uint32_t c, uint32_t b, const uint32_t* tl) {
  return tl[((c ^ b) & 0xffu) << 5] ^ (c >> 8);
}

__device__ __forceinline__ uint32_t crc_word(uint32_t c, uint32_t w, const uint32_t* tl) {
  c = crc_byte(c, w, tl);
  c = crc_byte(c, w >> 8, tl);
  c = crc_byte(c, w >> 16, tl);
  return crc_byte(c, w >> 24, tl);
}

// raw CRC of [p, p + n): bytes up to a 16-byte boundary, 64-byte blocks of four 16-byte loads, 16-byte loads, bytes
__device__ uint32_t raw_crc(const uint8_t* p, int64_t n, const uint32_t* tl) {
  uint32_t c = 0;
  int64_t head = (int64_t)((16 - ((uintptr_t)p & 15)) & 15);
  if (head > n) head = n;
  for (int64_t i = 0; i < head; ++i) c = crc_byte(c, __ldg(p + i), tl);
  p += head;
  n -= head;
  const uint4* q = reinterpret_cast<const uint4*>(p);
  for (; n >= 64; n -= 64, q += 4) {
    uint4 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = __ldg(q + k);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      c = crc_word(c, v[k].x, tl);
      c = crc_word(c, v[k].y, tl);
      c = crc_word(c, v[k].z, tl);
      c = crc_word(c, v[k].w, tl);
    }
  }
  for (; n >= 16; n -= 16, ++q) {
    const uint4 v = __ldg(q);
    c = crc_word(crc_word(crc_word(crc_word(c, v.x, tl), v.y, tl), v.z, tl), v.w, tl);
  }
  p = reinterpret_cast<const uint8_t*>(q);
  for (int64_t i = 0; i < n; ++i) c = crc_byte(c, __ldg(p + i), tl);
  return c;
}

__global__ void __launch_bounds__(kThreads) crc_rows_kernel(const uint8_t* __restrict__ base, int64_t rows,
                                                            int64_t row_bytes, int64_t row_stride, int64_t segs,
                                                            uint32_t len_term, uint32_t* __restrict__ out) {
  __shared__ uint32_t table[256 * 32];
  __shared__ uint32_t pw[64];
  fill_table(table, pw);
  const uint32_t* tl = table + (threadIdx.x & 31);
  const int64_t units = rows * segs;
  for (int64_t u = (int64_t)blockIdx.x * kThreads + threadIdx.x; u < units; u += (int64_t)gridDim.x * kThreads) {
    const int64_t r = u / segs, s = u - r * segs;
    const int64_t lo = s * kSeg, hi = lo + kSeg < row_bytes ? lo + kSeg : row_bytes;
    uint32_t c = raw_crc(base + r * row_stride + lo, hi - lo, tl);
    if (hi < row_bytes) c = mulmodp(c, xpow8((uint64_t)(row_bytes - hi), pw));
    if (s == 0) c ^= len_term;
    if (segs == 1) out[r] = c;
    else atomicXor(out + r, c);
  }
}

__global__ void __launch_bounds__(kThreads) crc_combine_kernel(const uint32_t* __restrict__ crcs, int64_t n, int64_t pad,
                                                               int64_t seg_bytes, uint32_t* __restrict__ out) {
  __shared__ uint32_t pw[64];
  __shared__ uint32_t part[kThreads / 32];
  if (threadIdx.x < 64) pw[threadIdx.x] = kPowDev.v[threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t k = xpow8((uint64_t)seg_bytes, pw);              // one leaf's bytes
  const int64_t j0 = (int64_t)blockIdx.x * kLeavesPerBlock + (int64_t)threadIdx.x * kRun;
  uint32_t acc = 0;
#pragma unroll
  for (int i = 0; i < kRun; ++i) {
    const int64_t leaf = j0 + i - pad;
    acc = mulmodp(acc, k) ^ (leaf >= 0 && leaf < n ? __ldg(crcs + leaf) : 0u);
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) k = mulmodp(k, k);             // kRun leaves
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t right = __shfl_down_sync(0xffffffffu, acc, o);
    acc = mulmodp(acc, k) ^ right;                           // meaningful on lanes that are multiples of 2 o
    k = mulmodp(k, k);
  }
  if (lane == 0) part[warp] = acc;
  __syncthreads();
  if (warp == 0) {
    acc = lane < kThreads / 32 ? part[lane] : 0u;
#pragma unroll
    for (int o = 1; o < kThreads / 32; o <<= 1) {
      const uint32_t right = __shfl_down_sync(0xffffffffu, acc, o);
      acc = mulmodp(acc, k) ^ right;
      k = mulmodp(k, k);
    }
    if (lane == 0) {
      const uint64_t after = (uint64_t)(gridDim.x - 1 - blockIdx.x) * (uint64_t)kLeavesPerBlock * (uint64_t)seg_bytes;
      atomicXor(out, mulmodp(acc, xpow8(after, pw)));
    }
  }
}

// The Keras output kernel's transpose (DESIGN.md §6l): a [k, Y] chunk of file rows <-> columns [col0, col0 + k) of the
// engine's [Y, ld] table.  32 x 32 tiles through shared memory (one padding word per row, so the column reads do not
// conflict), 32 x 8 threads, a grid-stride loop over the tiles; the element is moved as a uint32, so every bit survives.
constexpr int kTile = 32;
constexpr int kTileRows = 8;

__global__ void __launch_bounds__(kTile * kTileRows) rows_to_cols_kernel(const uint32_t* __restrict__ src, int64_t k,
                                                                          int64_t Y, uint32_t* __restrict__ dst,
                                                                          int64_t ld, int64_t col0) {
  __shared__ uint32_t tile[kTile][kTile + 1];
  const int64_t tiles_y = (Y + kTile - 1) / kTile, tiles = tiles_y * ((k + kTile - 1) / kTile);
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int64_t y0 = (t % tiles_y) * kTile, i0 = (t / tiles_y) * kTile;
#pragma unroll
    for (int r = 0; r < kTile; r += kTileRows) {              // read along y: src row i0 + ty + r
      const int64_t i = i0 + ty + r, y = y0 + tx;
      if (i < k && y < Y) tile[ty + r][tx] = __ldg(src + i * Y + y);
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < kTile; r += kTileRows) {              // write along i: dst row y0 + ty + r
      const int64_t y = y0 + ty + r, i = i0 + tx;
      if (i < k && y < Y) dst[y * ld + col0 + i] = tile[tx][ty + r];
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kTile * kTileRows) cols_to_rows_kernel(const uint32_t* __restrict__ src, int64_t ld,
                                                                          int64_t col0, int64_t k, int64_t Y,
                                                                          uint32_t* __restrict__ dst) {
  __shared__ uint32_t tile[kTile][kTile + 1];
  const int64_t tiles_y = (Y + kTile - 1) / kTile, tiles = tiles_y * ((k + kTile - 1) / kTile);
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int64_t y0 = (t % tiles_y) * kTile, i0 = (t / tiles_y) * kTile;
#pragma unroll
    for (int r = 0; r < kTile; r += kTileRows) {              // read along i: src row y0 + ty + r
      const int64_t y = y0 + ty + r, i = i0 + tx;
      if (i < k && y < Y) tile[ty + r][tx] = __ldg(src + y * ld + col0 + i);
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < kTile; r += kTileRows) {              // write along y: dst row i0 + ty + r
      const int64_t i = i0 + ty + r, y = y0 + tx;
      if (i < k && y < Y) dst[i * Y + y] = tile[tx][ty + r];
    }
    __syncthreads();
  }
}

int cfail(int code, const std::string& msg) {
  c2v::set_global_error(msg);
  return code;
}

int launch_check(const char* fn) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cfail(C2V_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(e));
  return C2V_OK;
}

int grid_for(int64_t units) {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  const int64_t want = (units + kThreads - 1) / kThreads;
  const int64_t cap = (int64_t)sms * 8;
  return (int)(want < cap ? want : cap);
}

}  // namespace

int c2v_crc32c_rows(const void* base, int64_t rows, int64_t row_bytes, int64_t row_stride, uint32_t* crc_out,
                    void* stream) {
  if (rows < 0 || row_bytes < 0 || (rows > 1 && row_stride < row_bytes))
    return cfail(C2V_ERR_INVALID, "c2v_crc32c_rows: need rows >= 0, row_bytes >= 0 and row_stride >= row_bytes");
  if (rows && (!crc_out || (row_bytes && !base)))
    return cfail(C2V_ERR_INVALID, "c2v_crc32c_rows: NULL argument");
  if (!rows) return C2V_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t segs = (row_bytes + kSeg - 1) / kSeg;
  if (segs != 1) {
    const cudaError_t e = cudaMemsetAsync(crc_out, 0, (size_t)rows * sizeof(uint32_t), s);
    if (e != cudaSuccess) return cfail(C2V_ERR_CUDA, std::string("c2v_crc32c_rows: ") + cudaGetErrorString(e));
  }
  if (!segs) return C2V_OK;                                  // the CRC of no bytes is 0
  const uint32_t len_term = mulmodp(0xFFFFFFFFu, xpow8((uint64_t)row_bytes, kPowHost.v)) ^ 0xFFFFFFFFu;
  crc_rows_kernel<<<grid_for(rows * segs), kThreads, 0, s>>>((const uint8_t*)base, rows, row_bytes, row_stride, segs,
                                                             len_term, crc_out);
  return launch_check("c2v_crc32c_rows");
}

int c2v_crc32c_combine(const uint32_t* crcs, int64_t n, int64_t seg_bytes, uint32_t* out, void* stream) {
  if (n < 0 || seg_bytes < 0) return cfail(C2V_ERR_INVALID, "c2v_crc32c_combine: need n >= 0 and seg_bytes >= 0");
  if (!out || (n && !crcs)) return cfail(C2V_ERR_INVALID, "c2v_crc32c_combine: NULL argument");
  cudaStream_t s = (cudaStream_t)stream;
  const cudaError_t e = cudaMemsetAsync(out, 0, sizeof(uint32_t), s);
  if (e != cudaSuccess) return cfail(C2V_ERR_CUDA, std::string("c2v_crc32c_combine: ") + cudaGetErrorString(e));
  if (!n) return C2V_OK;
  const int64_t blocks = (n + kLeavesPerBlock - 1) / kLeavesPerBlock;
  if (blocks > 0x7fffffff) return cfail(C2V_ERR_INVALID, "c2v_crc32c_combine: n too large");
  crc_combine_kernel<<<(unsigned)blocks, kThreads, 0, s>>>(crcs, n, blocks * kLeavesPerBlock - n, seg_bytes, out);
  return launch_check("c2v_crc32c_combine");
}

namespace {

// shared checks of the two transpose entry points; 0 = launch, 1 = nothing to move, < 0 = refused
int transpose_args(const char* fn, const void* src, int64_t k, int64_t Y, const void* dst, int64_t ld, int64_t col0) {
  if (k < 0 || Y < 0 || col0 < 0 || (k && Y && ld < col0 + k))
    return cfail(C2V_ERR_INVALID, std::string(fn) + ": need k >= 0, Y >= 0, col0 >= 0 and ld >= col0 + k");
  if (!k || !Y) return 1;
  if (!src || !dst) return cfail(C2V_ERR_INVALID, std::string(fn) + ": NULL argument");
  if (((uintptr_t)src | (uintptr_t)dst) & 3u)
    return cfail(C2V_ERR_INVALID, std::string(fn) + ": src and dst must be 4-byte aligned");
  return 0;
}

int transpose_grid(int64_t k, int64_t Y) {
  return grid_for(((Y + kTile - 1) / kTile) * ((k + kTile - 1) / kTile) * kThreads);
}

}  // namespace

int c2v_rows_to_cols(const float* src, int64_t k, int64_t Y, float* dst, int64_t ld, int64_t col0, void* stream) {
  const int rc = transpose_args("c2v_rows_to_cols", src, k, Y, dst, ld, col0);
  if (rc) return rc < 0 ? rc : C2V_OK;
  rows_to_cols_kernel<<<transpose_grid(k, Y), dim3(kTile, kTileRows), 0, (cudaStream_t)stream>>>(
      (const uint32_t*)src, k, Y, (uint32_t*)dst, ld, col0);
  return launch_check("c2v_rows_to_cols");
}

int c2v_cols_to_rows(const float* src, int64_t ld, int64_t col0, int64_t k, int64_t Y, float* dst, void* stream) {
  const int rc = transpose_args("c2v_cols_to_rows", src, k, Y, dst, ld, col0);
  if (rc) return rc < 0 ? rc : C2V_OK;
  cols_to_rows_kernel<<<transpose_grid(k, Y), dim3(kTile, kTileRows), 0, (cudaStream_t)stream>>>(
      (const uint32_t*)src, ld, col0, k, Y, (uint32_t*)dst);
  return launch_check("c2v_cols_to_rows");
}
