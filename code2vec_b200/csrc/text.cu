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

namespace c2v {
void set_global_error(const std::string& msg);     // engine.cu: the message c2v_last_error(NULL) returns
}

namespace {

// ---- exact unsigned integers of up to 256 bits (little-endian 32-bit words) -----------------------------------------
// The largest value the algorithm holds is below 2^194: a subnormal's scale is 2^151, its value times 10 stays below
// 10 * scale, and the high margin adds at most as much again.
constexpr int kWords = 8;

struct Big {
  uint32_t w[kWords];
  int n;            // words in use; w[n - 1] != 0 unless n == 0
};

__host__ __device__ inline void big_set(Big& a, uint64_t v) {
  for (int i = 0; i < kWords; ++i) a.w[i] = 0;
  a.w[0] = (uint32_t)v;
  a.w[1] = (uint32_t)(v >> 32);
  a.n = a.w[1] ? 2 : (a.w[0] ? 1 : 0);
}

__host__ __device__ inline void big_trim(Big& a) {
  while (a.n > 0 && a.w[a.n - 1] == 0) --a.n;
}

__host__ __device__ inline void big_pow2(Big& a, int e) {      // a = 2^e, 0 <= e < 32 * kWords
  big_set(a, 0);
  a.w[e / 32] = 1u << (e % 32);
  a.n = e / 32 + 1;
}

__host__ __device__ inline void big_shl(Big& a, int s) {       // a <<= s (s >= 0)
  if (a.n == 0 || s == 0) return;
  const int ws = s / 32, bs = s % 32;
  for (int i = kWords - 1; i >= 0; --i) {
    uint32_t v = 0;
    const int j = i - ws;
    if (j >= 0) {
      v = a.w[j] << bs;
      if (bs && j > 0) v |= a.w[j - 1] >> (32 - bs);
    }
    a.w[i] = v;
  }
  a.n = kWords;
  big_trim(a);
}

__host__ __device__ inline void big_mul_small(Big& a, uint32_t m) {
  uint64_t carry = 0;
  for (int i = 0; i < a.n; ++i) {
    const uint64_t p = (uint64_t)a.w[i] * m + carry;
    a.w[i] = (uint32_t)p;
    carry = p >> 32;
  }
  if (carry) a.w[a.n++] = (uint32_t)carry;
}

__host__ __device__ inline void big_mul_pow10(Big& a, int p) {  // a *= 10^p (p >= 0)
  for (; p >= 9; p -= 9) big_mul_small(a, 1000000000u);
  uint32_t m = 1;
  for (; p > 0; --p) m *= 10;
  if (m != 1) big_mul_small(a, m);
}

__host__ __device__ inline int big_cmp(const Big& a, const Big& b) {
  if (a.n != b.n) return a.n < b.n ? -1 : 1;
  for (int i = a.n - 1; i >= 0; --i)
    if (a.w[i] != b.w[i]) return a.w[i] < b.w[i] ? -1 : 1;
  return 0;
}

__host__ __device__ inline void big_add(Big& r, const Big& a, const Big& b) {
  const int n = a.n > b.n ? a.n : b.n;
  uint64_t carry = 0;
  for (int i = 0; i < n; ++i) {
    const uint64_t s = (uint64_t)(i < a.n ? a.w[i] : 0) + (i < b.n ? b.w[i] : 0) + carry;
    r.w[i] = (uint32_t)s;
    carry = s >> 32;
  }
  for (int i = n; i < kWords; ++i) r.w[i] = 0;
  r.n = n;
  if (carry) r.w[r.n++] = 1;
}

__host__ __device__ inline void big_sub(Big& a, const Big& b) {  // a -= b, a >= b
  int64_t borrow = 0;
  for (int i = 0; i < a.n; ++i) {
    const int64_t d = (int64_t)a.w[i] - (i < b.n ? b.w[i] : 0) - borrow;
    a.w[i] = (uint32_t)d;
    borrow = d < 0;
  }
  big_trim(a);
}

// a = a mod b and the quotient, for a < 10 * b
__host__ __device__ inline int big_divmod_digit(Big& a, const Big& b) {
  int q = 0;
  while (q < 9 && big_cmp(a, b) >= 0) {
    big_sub(a, b);
    ++q;
  }
  return q;
}

__host__ __device__ inline int clz32(uint32_t v) {
#ifdef __CUDA_ARCH__
  return __clz(v);
#else
  return __builtin_clz(v);
#endif
}

// ---- Dragon4, numpy's "unique" mode ---------------------------------------------------------------------------------
constexpr int kMaxDigits = 9;       // nine significant digits identify every float32

// The shortest digits of a finite, non-zero float32 magnitude (bits without the sign) and the decimal exponent of the
// first digit.  Returns the number of digits.
__host__ __device__ inline int dragon4(uint32_t bits, char* digits, int* exp10) {
  const uint32_t fexp = bits >> 23, fmant = bits & 0x7fffffu;
  uint32_t mant;
  int e, mant_bit;
  bool unequal;
  if (fexp) {
    mant = fmant | (1u << 23);
    e = (int)fexp - 127 - 23;
    mant_bit = 23;
    unequal = fexp != 1 && fmant == 0;    // the next float32 down is half as far away
  } else {
    mant = fmant;
    e = 1 - 127 - 23;
    mant_bit = 31 - clz32(mant);
    unequal = false;
  }
  // value / scale = the magnitude; margin_lo / scale and margin_hi / scale = the distances to the rounding interval's
  // ends (half an ulp below and above), everything scaled to integers
  Big value, scale, lo, hi;
  if (e >= 0) {
    big_set(value, mant);
    big_shl(value, e + (unequal ? 2 : 1));
    big_set(scale, unequal ? 4 : 2);
    big_pow2(lo, e);
  } else {
    big_set(value, (uint64_t)mant << (unequal ? 2 : 1));
    big_pow2(scale, -e + (unequal ? 2 : 1));
    big_set(lo, 1);
  }
  // first-digit estimate, exact or one too small (the correction below); computed as numpy computes it
  int k = (int)ceil((double)(mant_bit + e) * 0.30102999566398119521 - 0.69);
  if (k > 0) {
    big_mul_pow10(scale, k);
  } else if (k < 0) {
    big_mul_pow10(value, -k);
    big_mul_pow10(lo, -k);
  }
  if (big_cmp(value, scale) >= 0) {
    ++k;
  } else {
    big_mul_small(value, 10);
    big_mul_small(lo, 10);
  }
  hi = lo;
  if (unequal) big_shl(hi, 1);
  const bool even = (mant & 1) == 0;
  *exp10 = k - 1;

  int n = 0, digit = 0;
  bool low = false, high = false;
  Big top;
  for (;;) {
    digit = big_divmod_digit(value, scale);
    big_add(top, value, hi);
    // the digits so far, rounded down (low) or up (high), still name this float; an even mantissa owns the interval's
    // ends (round-to-even reads them back as this float), an odd one does not
    const int cl = big_cmp(value, lo), ch = big_cmp(top, scale);
    low = even ? cl <= 0 : cl < 0;
    high = even ? ch >= 0 : ch > 0;
    if (low || high || n + 1 == kMaxDigits) break;
    digits[n++] = (char)('0' + digit);
    big_mul_small(value, 10);
    big_mul_small(lo, 10);
    big_mul_small(hi, 10);
  }
  bool round_down = low;
  if (low == high) {                       // both ends reachable: the nearer one, ties to an even digit
    big_shl(value, 1);
    const int c = big_cmp(value, scale);
    round_down = c < 0 || (c == 0 && (digit & 1) == 0);
  }
  if (round_down) {
    digits[n++] = (char)('0' + digit);
  } else if (digit < 9) {
    digits[n++] = (char)('0' + digit + 1);
  } else {                                 // carry through the trailing nines
    for (;;) {
      if (n == 0) {
        digits[n++] = '1';
        *exp10 += 1;
        break;
      }
      if (digits[n - 1] != '9') {
        digits[n - 1] += 1;
        break;
      }
      --n;
    }
  }
  return n;
}

// str(np.float32(x)) into out (at least 16 bytes; the text is at most 15); returns its length.  Not NUL-terminated.
__host__ __device__ int format_f32(float x, char* out) {
  uint32_t bits;
  memcpy(&bits, &x, 4);
  const bool neg = bits >> 31;
  const uint32_t mag = bits & 0x7fffffffu;
  int p = 0;
  if (mag > 0x7f800000u) {
    out[0] = 'n'; out[1] = 'a'; out[2] = 'n';
    return 3;
  }
  if (neg) out[p++] = '-';
  if (mag == 0x7f800000u) {
    out[p++] = 'i'; out[p++] = 'n'; out[p++] = 'f';
    return p;
  }
  if (mag == 0) {
    out[p++] = '0'; out[p++] = '.'; out[p++] = '0';
    return p;
  }
  char d[kMaxDigits];
  int e10;
  const int n = dragon4(mag, d, &e10);
  const double a = fabs((double)x);
  if (a >= 1e-4 && a < 1e6) {               // positional: e10 in [-4, 5]
    if (e10 >= 0) {
      for (int i = 0; i <= e10; ++i) out[p++] = i < n ? d[i] : '0';
      out[p++] = '.';
      if (n > e10 + 1) {
        for (int i = e10 + 1; i < n; ++i) out[p++] = d[i];
      } else {
        out[p++] = '0';
      }
    } else {
      out[p++] = '0';
      out[p++] = '.';
      for (int i = 0; i < -e10 - 1; ++i) out[p++] = '0';
      for (int i = 0; i < n; ++i) out[p++] = d[i];
    }
    return p;
  }
  out[p++] = d[0];
  if (n > 1) {
    out[p++] = '.';
    for (int i = 1; i < n; ++i) out[p++] = d[i];
  }
  out[p++] = 'e';
  out[p++] = e10 < 0 ? '-' : '+';
  const int ae = e10 < 0 ? -e10 : e10;     // |e10| <= 45
  out[p++] = (char)('0' + ae / 10);
  out[p++] = (char)('0' + ae % 10);
  return p;
}

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
