// The native tensoriser's vocabulary hash table (native/batcher.cpp Vocab) in device memory, and its lookup: shared by
// the device reader (reader.cu) and the device predictor (predict.cu).  Internal linkage, as float_text.cuh.
#pragma once

#include <stdint.h>

namespace {

struct DevSlot {                  // native/batcher.cpp Vocab::Slot, byte for byte
  unsigned long long h;           // FNV-1a 64 of the word (0: empty slot)
  long long off;                  // offset of the word's bytes
  int32_t len, idx;
};
static_assert(sizeof(DevSlot) == 24, "slot layout of batcher.cpp");

struct DevVocab {
  const DevSlot* slots;
  const unsigned char* bytes;
  unsigned long long mask;
  int32_t oov, pad;
};

__device__ __forceinline__ unsigned long long fnv1a(const unsigned char* p, long long n) {
  unsigned long long h = 1469598103934665603ull;
  for (long long i = 0; i < n; ++i) { h ^= p[i]; h *= 1099511628211ull; }
  return h ? h : 1;
}

// batcher.cpp Vocab::lookup: linear probing from h & mask, the first slot with the same hash, length and bytes wins
__device__ int32_t lookup(const DevVocab& v, const unsigned char* p, long long n) {
  const unsigned long long h = fnv1a(p, n);
  for (unsigned long long i = h & v.mask;; i = (i + 1) & v.mask) {
    const DevSlot* s = v.slots + i;
    const unsigned long long sh = s->h;
    if (sh == 0) return v.oov;
    if (sh == h && (long long)s->len == n) {
      const unsigned char* w = v.bytes + s->off;
      long long k = 0;
      while (k < n && w[k] == p[k]) ++k;
      if (k == n) return s->idx;
    }
  }
}

}  // namespace
