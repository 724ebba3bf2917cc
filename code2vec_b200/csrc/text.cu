// Float32 text on the device (include/c2v_b200.h "Text of float32 matrices", DESIGN.md §6f): rows of a float32 matrix
// -> the lines the host writers produce (model_base._write_code_vectors, common.save_word2vec_file), byte for byte.
// Every value is written as numpy's str(np.float32(x)) writes it:
//   specials   : "nan" (any sign or payload), "inf", "-inf", "0.0", "-0.0"
//   positional : 1e-4 <= |x| < 1e6, compared exactly (the float32 nearest 1e-4 lies below it): "0.5", "999999.0",
//                "0.000100000005"; always a digit after the point
//   scientific : anything else: "1e+07", "1.5e+08", "1e-45"; no trailing ".0", exponent signed, at least two digits
//   digits     : Dragon4 in numpy's "unique" mode (Steele & White's free-format algorithm on exact big integers), with
//                numpy's choices: both ends of the rounding interval excluded whatever the mantissa's parity, the last
//                digit rounded to nearest against the remainder with ties to an even digit, and the margins unequal
//                below a power of two.  Where a shortest-round-trip algorithm would choose other digits, this is numpy.
// The formatter is __host__ __device__: c2v_selftest_format_floats runs it on the CPU so that it can be compared with
// numpy over all 2^32 bit patterns (tools/float_text_sweep.py).  Its output is at most 15 bytes.
//   format kernel : one warp per row; each lane formats a column of each group of 32, a warp scan of the lengths
//                   places the text (separator included) in the row's stage slot of cols * 16 bytes
//   scan kernel   : one block; each row's end offset (prefix + text), and how many rows fit the output buffer
//   copy kernel   : one warp per fitting row; the prefix and the staged text, written contiguously to the output
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <cub/block/block_scan.cuh>
#include <string>

#include "../../include/c2v_b200.h"
#include "float_text.cuh"

namespace c2v {
void set_global_error(const std::string& msg);     // engine.cu: the message c2v_last_error(NULL) returns
}

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kWarpsPerBlock = 8;
constexpr int kScanThreads = 256;

int tfail(int code, const std::string& msg) {
  c2v::set_global_error(msg);
  return code;
}

// row r's values, each followed by ' ' (the last by '\n'), packed at stage + r * cols * C2V_TEXT_VALUE_BYTES; its length
// into row_len[r]
__global__ void __launch_bounds__(kWarpsPerBlock * 32) format_rows_kernel(const float* __restrict__ x, long long rows,
                                                                          int cols, long long ld, char* __restrict__ stage,
                                                                          long long* __restrict__ row_len) {
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* xr = x + r * ld;
  char* sr = stage + r * (long long)cols * C2V_TEXT_VALUE_BYTES;
  long long base = 0;
  for (int c0 = 0; c0 < cols; c0 += 32) {
    const int c = c0 + lane;
    char buf[C2V_TEXT_VALUE_BYTES];
    int len = 0;
    if (c < cols) {
      len = format_f32(xr[c], buf);
      buf[len++] = c == cols - 1 ? '\n' : ' ';
    }
    int incl = len;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(kFull, incl, o);
      if (lane >= o) incl += v;
    }
    char* dst = sr + base + (incl - len);
    for (int i = 0; i < len; ++i) dst[i] = buf[i];
    base += __shfl_sync(kFull, incl, 31);
  }
  if (lane == 0) row_len[r] = base;
}

// row_end[r] = the end of row r in the output (its prefix and text, rows back to back; on entry row_end[r] holds the
// text's length); rows_done = the rows that end within out_cap (a prefix of the rows: the ends grow)
__global__ void __launch_bounds__(kScanThreads) scan_rows_kernel(long long rows, const long long* __restrict__ prefix_off,
                                                                 long long* __restrict__ row_end, long long out_cap,
                                                                 long long* __restrict__ rows_done) {
  using Scan = cub::BlockScan<long long, kScanThreads>;
  __shared__ typename Scan::TempStorage tmp;
  long long carry = 0, done = 0;
  for (long long r0 = 0; r0 < rows; r0 += kScanThreads) {
    const long long r = r0 + threadIdx.x;
    long long len = 0;
    if (r < rows) len = row_end[r] + (prefix_off ? prefix_off[r + 1] - prefix_off[r] : 0);
    long long incl, total;
    Scan(tmp).InclusiveSum(len, incl, total);
    const long long end = carry + incl;
    if (r < rows) row_end[r] = end;
    done += __syncthreads_count(r < rows && end <= out_cap);     // also the barrier before tmp is used again
    carry += total;
  }
  if (threadIdx.x == 0) *rows_done = done;
}

// rows [0, *rows_done): the prefix, then the staged text, at out + the row's start
__global__ void __launch_bounds__(kWarpsPerBlock * 32) copy_rows_kernel(long long rows, int cols,
                                                                        const char* __restrict__ prefix,
                                                                        const long long* __restrict__ prefix_off,
                                                                        const char* __restrict__ stage,
                                                                        const long long* __restrict__ row_end,
                                                                        const long long* __restrict__ rows_done,
                                                                        char* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (r >= rows || r >= *rows_done) return;
  char* dst = out + (r ? row_end[r - 1] : 0);
  long long np = 0;
  if (prefix_off) {
    const long long p0 = prefix_off[r];
    np = prefix_off[r + 1] - p0;
    for (long long i = lane; i < np; i += 32) dst[i] = prefix[p0 + i];
  }
  const char* src = stage + r * (long long)cols * C2V_TEXT_VALUE_BYTES;
  const long long nt = row_end[r] - (r ? row_end[r - 1] : 0) - np;
  for (long long i = lane; i < nt; i += 32) dst[np + i] = src[i];
}

}  // namespace

int c2v_text_format_rows(const float* x, int64_t rows, int32_t cols, int64_t ld, const char* prefix,
                         const int64_t* prefix_off, void* stage, size_t stage_bytes, char* out, int64_t out_cap,
                         int64_t* row_end, int64_t* rows_done, void* stream) {
  if (rows < 0 || cols < 1 || ld < cols || out_cap < 0)
    return tfail(C2V_ERR_INVALID, "c2v_text_format_rows: need rows >= 0, cols >= 1, ld >= cols and out_cap >= 0");
  if (!rows_done || (rows && (!x || !stage || !out || !row_end)) || (!prefix != !prefix_off))
    return tfail(C2V_ERR_INVALID, "c2v_text_format_rows: NULL argument (prefix and prefix_off go together)");
  if ((uint64_t)rows * (uint64_t)cols * C2V_TEXT_VALUE_BYTES > stage_bytes)
    return tfail(C2V_ERR_INVALID, "c2v_text_format_rows: stage_bytes below rows * cols * C2V_TEXT_VALUE_BYTES");
  cudaStream_t s = (cudaStream_t)stream;
  const long long grid = (rows + kWarpsPerBlock - 1) / kWarpsPerBlock;
  if (rows) {
    format_rows_kernel<<<(unsigned)grid, kWarpsPerBlock * 32, 0, s>>>(x, rows, cols, ld, (char*)stage,
                                                                       (long long*)row_end);
  }
  scan_rows_kernel<<<1, kScanThreads, 0, s>>>(rows, (const long long*)prefix_off, (long long*)row_end, out_cap,
                                              (long long*)rows_done);
  if (rows) {
    copy_rows_kernel<<<(unsigned)grid, kWarpsPerBlock * 32, 0, s>>>(rows, cols, prefix, (const long long*)prefix_off,
                                                                     (const char*)stage, (const long long*)row_end,
                                                                     (const long long*)rows_done, out);
  }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return tfail(C2V_ERR_CUDA, std::string("c2v_text_format_rows: ") + cudaGetErrorString(e));
  return C2V_OK;
}

int c2v_selftest_format_floats(const float* x, int64_t n, char* out, int32_t* len) {
  if (n < 0 || (n && (!x || !out || !len)))
    return tfail(C2V_ERR_INVALID, "c2v_selftest_format_floats: NULL argument or negative count");
  for (int64_t i = 0; i < n; ++i) {
    char* o = out + i * C2V_TEXT_VALUE_BYTES;
    len[i] = format_f32(x[i], o);
    for (int j = len[i]; j < C2V_TEXT_VALUE_BYTES; ++j) o[j] = 0;
  }
  return C2V_OK;
}
