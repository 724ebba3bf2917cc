// str(np.float32(x)) on the host and the device: exact big integers and numpy's Dragon4 (text.cu, DESIGN.md §6f), shared
// by the text writer (text.cu) and the predict formatter (predict.cu).  Everything here has internal linkage: each
// translation unit that includes it gets its own copy, so the kernels that call it compile as they did when it lived in
// text.cu.
#pragma once

#include <math.h>
#include <stdint.h>
#include <string.h>

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

// ---- '%f' % float(x): six decimals of the exact binary value, ties to even ----------------------------------------
constexpr int kFixedBytes = 48;     // "-" + 39 integer digits (FLT_MAX < 10^39) + "." + 6 decimals

// a = a / d, returns a mod d (d > 0)
__host__ __device__ inline uint32_t big_divmod_small(Big& a, uint32_t d) {
  uint64_t rem = 0;
  for (int i = a.n - 1; i >= 0; --i) {
    const uint64_t cur = (rem << 32) | a.w[i];
    a.w[i] = (uint32_t)(cur / d);
    rem = cur % d;
  }
  big_trim(a);
  return (uint32_t)rem;
}

// Python's '%f' % float(x) for a float32 x into out (at least kFixedBytes bytes); returns its length.  Not NUL-terminated.
// "nan" for every NaN, "inf" / "-inf", otherwise the value times 10^6 rounded to an integer (half to even, on the exact
// binary value), printed with six decimals and the sign of x ("-0.000000" for -0.0 and for negatives that round to 0).
__host__ __device__ inline int format_fixed6(float x, char* out) {
  uint32_t bits;
  memcpy(&bits, &x, 4);
  const uint32_t mag = bits & 0x7fffffffu;
  int p = 0;
  if (mag > 0x7f800000u) {
    out[0] = 'n'; out[1] = 'a'; out[2] = 'n';
    return 3;
  }
  if (bits >> 31) out[p++] = '-';
  if (mag == 0x7f800000u) {
    out[p++] = 'i'; out[p++] = 'n'; out[p++] = 'f';
    return p;
  }
  const uint32_t fexp = mag >> 23, fmant = mag & 0x7fffffu;
  const uint32_t mant = fexp ? (fmant | (1u << 23)) : fmant;
  const int e = fexp ? (int)fexp - 150 : -149;          // |x| = mant * 2^e
  Big n;                                                // round(|x| * 10^6)
  if (e >= 0) {
    big_set(n, mant);
    big_shl(n, e);
    big_mul_pow10(n, 6);
  } else {
    const uint64_t num = (uint64_t)mant * 1000000u;    // < 2^44
    const int k = -e;
    uint64_t q = 0;
    if (k < 64) {
      q = num >> k;
      const uint64_t rem = num - (q << k), half = 1ull << (k - 1);
      if (rem > half || (rem == half && (q & 1))) ++q;
    }                                                   // k >= 64: num < 2^44 < half, rounds to 0
    big_set(n, q);
  }
  const uint32_t frac = big_divmod_small(n, 1000000u);
  char digits[40];
  int nd = 0;
  while (n.n > 0) {                                     // the integer part, nine digits at a time from the bottom
    uint32_t chunk = big_divmod_small(n, 1000000000u);
    for (int i = 0; i < 9 && (n.n > 0 || chunk); ++i) {
      digits[nd++] = (char)('0' + chunk % 10);
      chunk /= 10;
    }
  }
  if (nd == 0) digits[nd++] = '0';
  while (nd > 0) out[p++] = digits[--nd];
  out[p++] = '.';
  uint32_t f = frac;
  for (int i = 5; i >= 0; --i) {
    out[p + i] = (char)('0' + f % 10);
    f /= 10;
  }
  return p + 6;
}

}  // namespace
