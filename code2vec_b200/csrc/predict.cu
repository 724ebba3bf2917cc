// Device predict (include/c2v_b200.h "Device predict", DESIGN.md §6i): extractor output in device memory -> the model
// input rows of its methods, and the text `python -m code2vec_b200 --predict` prints for them, byte for byte what the host
// route (__main__.print_predictions) prints.  ASCII input only; the caller routes anything else through the host.
//   chunk     : one chunk of whole lines at a time.  Line ends (cub select: '\n', and a lone '\r' under universal
//               newlines; a "\r\n" ends at its '\n' and the '\r' goes with the rstrip), then one thread per line: rstrip,
//               the name field, the first max_contexts non-empty fields, each split into exactly three parts, each
//               path's key; kind per line (skipped, method, malformed, key the table cannot hold).  Over all chunks,
//               every key's last writer (largest file offset) goes into a hash table, and then, chunk by chunk again,
//               the winners' path texts into an arena, so a chunk's methods can print paths from any other chunk
//   rows      : one thread per method finds its kept contexts, one thread per slot hashes, looks up and masks
//   rank      : one block per method: first occurrence and last value of every (token, key, token) triple, then the
//               stable descending order of the distinct triples' values (all-NaN rows keep first-occurrence order), top 10
//   format    : one thread per method writes its block (length pass, scan, write pass) with format_fixed6 and format_f32
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>
#include <string>

#include "../../include/c2v_b200.h"
#include "float_text.cuh"
#include "vocab_lookup.cuh"

namespace c2v {
void set_global_error(const std::string& msg);     // engine.cu: the message c2v_last_error(NULL) returns
}

namespace {

constexpr int kThreads = 256;
constexpr int kTopContexts = 10;                   // __main__.SHOW_TOP_CONTEXTS

int pfail(int code, const std::string& msg) {
  c2v::set_global_error(msg);
  return code;
}
int pcuda(const char* fn, cudaError_t e) { return pfail(C2V_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(e)); }
#define PCHECK(fn, expr)                         \
  do {                                           \
    cudaError_t _c = (expr);                     \
    if (_c != cudaSuccess) return pcuda(fn, _c); \
  } while (0)

struct Buf {
  void* p = nullptr;
  size_t bytes = 0;
};

// ---- keys -----------------------------------------------------------------------------------------------------------
// str.rstrip() on ASCII: space, \t, \n, \v, \f, \r and \x1c-\x1f
__device__ __forceinline__ bool py_space(unsigned char c) { return c == ' ' || (c >= 9 && c <= 13) || (c >= 0x1c && c <= 0x1f); }
__device__ __forceinline__ bool digit(unsigned char c) { return (unsigned char)(c - '0') < 10; }

// A path's key as an int32 (the text of the key is its decimal): Java's String.hashCode of the path, or the path itself
// when it is -?[0-9]+ (__main__._looks_hashed).  Returns false for a numeric path that is not the canonical decimal of an
// int32 ("007", "-0", "2147483648"): its key is text no hash can print, which the caller leaves to the host route.
__device__ bool key_code(const unsigned char* s, long long n, int32_t* code) {
  const long long i0 = n > 0 && s[0] == '-' ? 1 : 0;
  bool numeric = i0 < n;
  for (long long i = i0; i < n && numeric; ++i) numeric = digit(s[i]);
  if (!numeric) {
    uint32_t h = 0;
    for (long long i = 0; i < n; ++i) h = h * 31u + s[i];
    *code = (int32_t)h;
    return true;
  }
  const long long len = n - i0;
  if (len > 10 || (len > 1 && s[i0] == '0') || (i0 && s[i0] == '0')) return false;
  unsigned long long v = 0;
  for (long long i = i0; i < n; ++i) v = v * 10 + (s[i] - '0');
  if (v > (i0 ? 2147483648ull : 2147483647ull)) return false;
  *code = (int32_t)(uint32_t)(i0 ? 0ull - v : v);
  return true;
}

__device__ int decimal(int32_t v, unsigned char* out) {     // str(v), at most 11 bytes
  int p = 0;
  unsigned int u = (unsigned int)v;
  if (v < 0) {
    out[p++] = '-';
    u = 0u - u;
  }
  char d[10];
  int nd = 0;
  do {
    d[nd++] = (char)('0' + u % 10);
    u /= 10;
  } while (u);
  while (nd) out[p++] = d[--nd];
  return p;
}

// ---- the last-writer table: key -> the path text of the last context with that key --------------------------------
// A slot holds the key (code + 2^32; 0: empty) and (file offset << 20 | length) of the key's path with the largest file
// offset so far (atomicMax, so the winner does not depend on atomic order).  Once every chunk has been recorded, the
// winners' texts are copied into an arena, chunk by chunk, and the formatter reads them from there.
constexpr int kLenBits = 20;                       // paths of 1 MB or more go to the host route
constexpr unsigned long long kLenMask = (1ull << kLenBits) - 1;

struct Unhash {
  unsigned long long* key;
  unsigned long long* val;
  unsigned long long mask;
  unsigned long long* used;    // occupied slots
  const long long* arena_off;  // per slot, once sealed
  const char* arena;
};

__device__ __forceinline__ unsigned long long slot_of(int32_t code, unsigned long long mask) {
  unsigned long long x = (uint32_t)code;
  x ^= x >> 16;
  x *= 0x45d9f3b3335b369ull;
  x ^= x >> 31;
  return x & mask;
}

__device__ void unhash_put(const Unhash& u, unsigned long long k, unsigned long long v) {
  for (unsigned long long i = slot_of((int32_t)(uint32_t)k, u.mask);; i = (i + 1) & u.mask) {
    const unsigned long long prev = atomicCAS(u.key + i, 0ull, k);
    if (prev == 0 || prev == k) {
      if (prev == 0) atomicAdd(u.used, 1ull);
      atomicMax(u.val + i, v);
      return;
    }
  }
}

__device__ __forceinline__ unsigned long long key_of(int32_t code) { return (unsigned long long)(uint32_t)code + (1ull << 32); }

__device__ long long unhash_slot(const Unhash& u, int32_t code) {
  const unsigned long long k = key_of(code);
  for (unsigned long long i = slot_of(code, u.mask);; i = (i + 1) & u.mask) {
    const unsigned long long cur = u.key[i];
    if (cur == 0) return -1;
    if (cur == k) return (long long)i;
  }
}

__global__ void __launch_bounds__(kThreads) rehash_kernel(const unsigned long long* __restrict__ key,
                                                          const unsigned long long* __restrict__ val,
                                                          unsigned long long slots, Unhash nu) {
  const unsigned long long i = (unsigned long long)blockIdx.x * kThreads + threadIdx.x;
  if (i < slots && key[i]) unhash_put(nu, key[i], val[i]);
}

__global__ void __launch_bounds__(kThreads) arena_len_kernel(const unsigned long long* __restrict__ key,
                                                             const unsigned long long* __restrict__ val,
                                                             unsigned long long slots, long long* __restrict__ len) {
  const unsigned long long i = (unsigned long long)blockIdx.x * kThreads + threadIdx.x;
  if (i < slots) len[i] = key[i] ? (long long)(val[i] & kLenMask) : 0;
}

// the winners whose path lies in this chunk [base, base + n) copy it into the arena
__global__ void __launch_bounds__(kThreads) arena_copy_kernel(const unsigned char* __restrict__ t, long long base, long long n,
                                                              const unsigned long long* __restrict__ key,
                                                              const unsigned long long* __restrict__ val,
                                                              unsigned long long slots,
                                                              const long long* __restrict__ arena_off,
                                                              char* __restrict__ arena) {
  const unsigned long long i = (unsigned long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= slots || !key[i]) return;
  const long long off = (long long)(val[i] >> kLenBits) - base, len = (long long)(val[i] & kLenMask);
  if (off < 0 || off >= n) return;
  for (long long j = 0; j < len; ++j) arena[arena_off[i] + j] = (char)t[off + j];
}

// ---- load: line index and the per-line scan -------------------------------------------------------------------------
struct IsLineEnd {
  const unsigned char* t;
  long long n;
  int universal;
  __device__ bool operator()(long long p) const {
    const unsigned char c = t[p];
    return c == '\n' || (universal && c == '\r' && (p + 1 == n || t[p + 1] != '\n'));
  }
};

struct LineEndCount {
  IsLineEnd is;
  __device__ long long operator()(long long p) const { return is(p) ? 1 : 0; }
};

enum LineKind : int32_t { kSkipped = 0, kMethod = 1, kMalformed = 2, kOddKey = 3 };

struct LineArgs {
  const unsigned char* t;
  long long n;
  const long long* ends;       // [n_ends] line terminators
  long long n_ends, n_lines;
  int C;
  long long* lo;               // [n_lines] the rstripped line [lo, hi)
  long long* hi;
  int32_t* kind;               // [n_lines]
  int32_t* kept;               // [n_lines] contexts kept
  Unhash u;
  int insert;                  // 0: scan only; 1: record every kept context's key in the table
  long long base;              // the chunk's offset in the file
};

__global__ void __launch_bounds__(kThreads) lines_kernel(const __grid_constant__ LineArgs a) {
  const long long l = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (l >= a.n_lines) return;
  const unsigned char* t = a.t;
  const long long lo = l ? a.ends[l - 1] + 1 : 0;
  long long hi = l < a.n_ends ? a.ends[l] : a.n;
  while (hi > lo && py_space(t[hi - 1])) --hi;
  long long p = lo;
  while (p < hi && t[p] != ' ') ++p;
  int32_t kind = p > lo ? kMethod : kSkipped;
  int kept = 0;
  while (kind == kMethod && p < hi && kept < a.C) {
    const long long fs = ++p;                 // p was on a space
    while (p < hi && t[p] != ' ') ++p;
    if (p == fs) continue;
    long long c1 = -1, c2 = -1;
    int commas = 0;
    for (long long q = fs; q < p; ++q) {
      if (t[q] == ',') {
        if (commas == 0) c1 = q;
        else if (commas == 1) c2 = q;
        ++commas;
      }
    }
    if (commas != 2) {
      kind = kMalformed;
      break;
    }
    int32_t code;
    if (!key_code(t + c1 + 1, c2 - c1 - 1, &code) || (unsigned long long)(c2 - c1 - 1) > kLenMask) {
      kind = kOddKey;
      break;
    }
    if (a.insert) unhash_put(a.u, key_of(code), (unsigned long long)(a.base + c1 + 1) << kLenBits | (c2 - c1 - 1));
    ++kept;
  }
  a.lo[l] = lo;
  a.hi[l] = hi;
  a.kind[l] = kind;
  a.kept[l] = kept;
}

// ---- rows ------------------------------------------------------------------------------------------------------------
struct Slot {                  // one context slot of a batch row; fs < 0: padding
  long long fs, c1, c2, fe;
};

struct RowsArgs {
  const unsigned char* t;
  const long long* line;       // [n] the rows' line numbers
  const long long* lo;
  const long long* hi;
  int n, C;
  Slot* slots;                 // [n, C]
  long long* name;             // [n, 2] the name field
  DevVocab tok, path;
  int32_t *src, *pth, *tgt;
  float* mask;
  int32_t* code;               // [n, C] key code
  unsigned long long* fp;      // [n, C] hash of the triple's text (0 for padding)
};

__global__ void __launch_bounds__(kThreads) split_kernel(const __grid_constant__ RowsArgs a) {
  const int r = blockIdx.x * kThreads + threadIdx.x;
  if (r >= a.n) return;
  const unsigned char* t = a.t;
  const long long l = a.line[r], lo = a.lo[l], hi = a.hi[l];
  long long p = lo;
  while (p < hi && t[p] != ' ') ++p;
  a.name[2 * r] = lo;
  a.name[2 * r + 1] = p;
  Slot* s = a.slots + (long long)r * a.C;
  int kept = 0;
  while (p < hi && kept < a.C) {
    const long long fs = ++p;
    while (p < hi && t[p] != ' ') ++p;
    if (p == fs) continue;
    long long c1 = fs;
    while (t[c1] != ',') ++c1;
    long long c2 = c1 + 1;
    while (t[c2] != ',') ++c2;
    s[kept++] = Slot{fs, c1, c2, p};
  }
  for (int c = kept; c < a.C; ++c) s[c] = Slot{-1, 0, 0, 0};
}

__device__ __forceinline__ unsigned long long fnv_more(unsigned long long h, const unsigned char* p, long long n) {
  for (long long i = 0; i < n; ++i) {
    h ^= p[i];
    h *= 1099511628211ull;
  }
  return h;
}

__global__ void __launch_bounds__(kThreads) lookup_kernel(const __grid_constant__ RowsArgs a) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= (long long)a.n * a.C) return;
  const Slot s = a.slots[i];
  if (s.fs < 0) {
    a.src[i] = a.tok.pad;
    a.pth[i] = a.path.pad;
    a.tgt[i] = a.tok.pad;
    a.mask[i] = 0.f;
    a.code[i] = 0;
    a.fp[i] = 0;
    return;
  }
  const unsigned char* t = a.t;
  int32_t code = 0;
  key_code(t + s.c1 + 1, s.c2 - s.c1 - 1, &code);
  unsigned char key[12];
  const int kl = decimal(code, key);
  const int32_t x = lookup(a.tok, t + s.fs, s.c1 - s.fs);
  const int32_t y = lookup(a.path, key, kl);
  const int32_t z = lookup(a.tok, t + s.c2 + 1, s.fe - s.c2 - 1);
  a.src[i] = x;
  a.pth[i] = y;
  a.tgt[i] = z;
  a.mask[i] = (x != a.tok.pad || z != a.tok.pad || y != a.path.pad) ? 1.f : 0.f;
  a.code[i] = code;
  unsigned long long h = fnv_more(1469598103934665603ull, t + s.fs, s.c1 - s.fs);
  h = fnv_more(h, key, kl);
  h = fnv_more(h ^ 0xff, t + s.c2 + 1, s.fe - s.c2 - 1);
  a.fp[i] = h | 1;
}

// ---- rank --------------------------------------------------------------------------------------------------------------
struct RankArgs {
  const unsigned char* t;
  int n, C;
  const Slot* slots;
  const int32_t* code;
  const unsigned long long* fp;
  const float* attn;           // [n, C]
  int32_t* top;                // [n, 10] the entries' first slots, -1 past the last
  float* top_val;              // [n, 10] their values
  int32_t* bad_row;            // the lowest row whose attention is NaN in some distinct triples only
};

__device__ bool same_bytes(const unsigned char* t, long long a0, long long a1, long long b0, long long b1) {
  if (a1 - a0 != b1 - b0) return false;
  for (long long i = 0; i < a1 - a0; ++i)
    if (t[a0 + i] != t[b0 + i]) return false;
  return true;
}

__device__ __forceinline__ bool same_triple(const RankArgs& a, long long i, long long j) {
  if (a.fp[i] != a.fp[j]) return false;
  if (a.fp[i] == 0) return true;                      // both padding
  if (a.code[i] != a.code[j]) return false;
  const Slot x = a.slots[i], y = a.slots[j];
  return same_bytes(a.t, x.fs, x.c1, y.fs, y.c1) && same_bytes(a.t, x.c2 + 1, x.fe, y.c2 + 1, y.fe);
}

// dynamic shared memory: C floats (each distinct triple's value at its first slot) and C flags (first occurrence)
__global__ void __launch_bounds__(kThreads) rank_kernel(const __grid_constant__ RankArgs a) {
  extern __shared__ float sm[];
  float* val = sm;
  unsigned char* first = reinterpret_cast<unsigned char*>(sm + a.C);
  const int r = blockIdx.x, C = a.C;
  const long long base = (long long)r * C;
  int any_nan = 0, any_num = 0;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    bool f = true;
    int last = c;
    for (int d = 0; d < C; ++d) {
      if (d == c || !same_triple(a, base + c, base + d)) continue;
      if (d < c) {
        f = false;
        break;
      }
      last = d;
    }
    first[c] = f;
    if (f) {
      val[c] = a.attn[base + last];
      if (isnan(val[c])) any_nan = 1;
      else any_num = 1;
    }
  }
  if (threadIdx.x < kTopContexts) a.top[r * kTopContexts + threadIdx.x] = -1;
  any_nan = __syncthreads_or(any_nan);
  any_num = __syncthreads_or(any_num);
  if (any_nan && any_num) {
    if (threadIdx.x == 0) atomicMin(a.bad_row, r);
    return;
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    if (!first[c]) continue;
    const float v = val[c];
    int rank = 0;
    for (int d = 0; d < C && rank < kTopContexts; ++d) {
      if (!first[d] || d == c) continue;
      rank += any_nan ? d < c : (val[d] > v || (val[d] == v && d < c));
    }
    if (rank < kTopContexts) {
      a.top[r * kTopContexts + rank] = c;
      a.top_val[r * kTopContexts + rank] = v;
    }
  }
}

// ---- format ------------------------------------------------------------------------------------------------------------
struct FormatArgs {
  const unsigned char* t;
  int n, C, k, D;
  const long long* name;
  const Slot* slots;
  const int32_t* code;
  const int32_t* top;
  const float* top_val;
  const int32_t* idx;          // [n, k] top-k target ids
  const float* val;            // [n, k] their scores
  const float* cv;             // [n, D] code vectors, or NULL
  const char* repr;            // str(word.split("|")) of every target word
  const long long* repr_off;
  int n_words, oov;
  Unhash u;
  long long* row_end;          // [n] lengths, then (after the scan) ends
  char* out;
  long long cap;
  const int32_t* bad_row;
};

struct Emit {
  char* o;
  long long len;
  __device__ void put(const char* s, long long n) {
    if (o)
      for (long long i = 0; i < n; ++i) o[len + i] = s[i];
    len += n;
  }
  template <int N>
  __device__ void put(const char (&s)[N]) { put(s, N - 1); }
};

__device__ long long emit_block(const FormatArgs& a, int r, char* o) {
  Emit e{o, 0};
  const char* t = reinterpret_cast<const char*>(a.t);
  char num[kFixedBytes];
  e.put("Original name:\t");
  e.put(t + a.name[2 * r], a.name[2 * r + 1] - a.name[2 * r]);
  e.put("\n");
  for (int j = 0; j < a.k; ++j) {
    const int32_t id = a.idx[(long long)r * a.k + j];
    if (id < 0 || id >= a.n_words || id == a.oov) continue;      // lookup_word maps unknown ids to the OOV word
    e.put("\t(");
    e.put(num, format_fixed6(a.val[(long long)r * a.k + j], num));
    e.put(") predicted: ");
    e.put(a.repr + a.repr_off[id], a.repr_off[id + 1] - a.repr_off[id]);
    e.put("\n");
  }
  e.put("Attention:\n");
  for (int j = 0; j < kTopContexts; ++j) {
    const int c = a.top[r * kTopContexts + j];
    if (c < 0) break;
    const long long i = (long long)r * a.C + c;
    const Slot s = a.slots[i];
    if (s.fs < 0) continue;                          // the padding triple: its key is no path's
    const long long sl = unhash_slot(a.u, a.code[i]);
    const long long p0 = a.u.arena_off[sl], plen = (long long)(a.u.val[sl] & kLenMask);
    e.put(num, format_fixed6(a.top_val[r * kTopContexts + j], num));
    e.put("\tcontext: ");
    e.put(t + s.fs, s.c1 - s.fs + 1);                // token1 and its comma
    e.put(a.u.arena + p0, plen);
    e.put(t + s.c2, s.fe - s.c2);                    // the comma and token2
    e.put("\n");
  }
  if (a.cv) {
    e.put("Code vector:\n");
    for (int j = 0; j < a.D; ++j) {
      if (j) e.put(" ");
      e.put(num, format_f32(a.cv[(long long)r * a.D + j], num));
    }
    e.put("\n");
  }
  return e.len;
}

__global__ void __launch_bounds__(kThreads) block_len_kernel(const __grid_constant__ FormatArgs a) {
  const int r = blockIdx.x * kThreads + threadIdx.x;
  if (r < a.n) a.row_end[r] = emit_block(a, r, nullptr);
}

__global__ void __launch_bounds__(kThreads) block_write_kernel(const __grid_constant__ FormatArgs a) {
  const int r = blockIdx.x * kThreads + threadIdx.x;
  if (r >= a.n || a.row_end[a.n - 1] > a.cap || *a.bad_row < a.n) return;
  emit_block(a, r, a.out + (r ? a.row_end[r - 1] : 0));
}

unsigned grid_of(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

}  // namespace

struct c2v_pred {
  int device = 0;
  int C = 0;
  DevVocab tok{}, path{};
  Buf text, ends, lo, hi, kind, kept, key, val, arena_off, arena, scalars, tmp, repr, repr_off;
  Buf line, slots, name, code, fp, top, top_val, row_end;
  long long n_text = 0, n_lines = 0, n_rows = 0;
  int n_words = 0, oov = 0;
  unsigned long long mask = 0;     // table slots - 1
  bool sealed = false;             // the arena holds every key's path
  size_t held = 0, peak = 0;
};

namespace {

int grow(c2v_pred* h, Buf& b, size_t bytes, const char* fn) {
  if (bytes <= b.bytes && b.p) return C2V_OK;
  if (b.p) {
    cudaFree(b.p);
    h->held -= b.bytes;
    b.p = nullptr;
    b.bytes = 0;
  }
  if (bytes < 256) bytes = 256;
  PCHECK(fn, cudaMalloc(&b.p, bytes));
  b.bytes = bytes;
  h->held += bytes;
  if (h->held > h->peak) h->peak = h->held;
  return C2V_OK;
}

template <class T>
T* P(const Buf& b) { return reinterpret_cast<T*>(b.p); }

DevVocab dev_vocab(const c2v_reader_vocab& v) {
  return DevVocab{reinterpret_cast<const DevSlot*>(v.slots), reinterpret_cast<const unsigned char*>(v.bytes), v.mask, v.oov,
                  v.pad};
}

}  // namespace

int c2v_pred_create(int device, int32_t max_contexts, const c2v_reader_vocab* tok, const c2v_reader_vocab* path,
                    c2v_pred** out) {
  if (!out || !tok || !path) return pfail(C2V_ERR_INVALID, "c2v_pred_create: NULL argument");
  *out = nullptr;
  if (max_contexts < 1 || max_contexts > 4096) return pfail(C2V_ERR_INVALID, "c2v_pred_create: max_contexts not in [1, 4096]");
  PCHECK("c2v_pred_create", cudaSetDevice(device));
  c2v_pred* h = new c2v_pred;
  h->device = device;
  h->C = max_contexts;
  h->tok = dev_vocab(*tok);
  h->path = dev_vocab(*path);
  *out = h;
  return C2V_OK;
}

void c2v_pred_destroy(c2v_pred* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  for (Buf* b : {&h->text, &h->ends, &h->lo, &h->hi, &h->kind, &h->kept, &h->key, &h->val, &h->arena_off, &h->arena,
                 &h->scalars, &h->tmp, &h->repr,
                 &h->repr_off, &h->line, &h->slots, &h->name, &h->code, &h->fp, &h->top, &h->top_val, &h->row_end})
    if (b->p) cudaFree(b->p);
  delete h;
}

size_t c2v_pred_device_bytes(const c2v_pred* h) { return h ? h->peak : 0; }

int c2v_pred_set_targets(c2v_pred* h, int32_t n_words, const char* repr, const int64_t* repr_off, int32_t oov, void* stream) {
  static const char* fn = "c2v_pred_set_targets";
  if (!h || !repr || !repr_off || n_words < 1) return pfail(C2V_ERR_INVALID, "c2v_pred_set_targets: NULL argument or no words");
  PCHECK(fn, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  if ((rc = grow(h, h->repr, (size_t)repr_off[n_words], fn)) || (rc = grow(h, h->repr_off, (size_t)(n_words + 1) * 8, fn)))
    return rc;
  PCHECK(fn, cudaMemcpyAsync(h->repr.p, repr, (size_t)repr_off[n_words], cudaMemcpyHostToDevice, s));
  PCHECK(fn, cudaMemcpyAsync(h->repr_off.p, repr_off, (size_t)(n_words + 1) * 8, cudaMemcpyHostToDevice, s));
  PCHECK(fn, cudaStreamSynchronize(s));
  h->n_words = n_words;
  h->oov = oov;
  return C2V_OK;
}

namespace {

Unhash table_of(c2v_pred* h) {
  return Unhash{P<unsigned long long>(h->key), P<unsigned long long>(h->val), h->mask, P<unsigned long long>(h->scalars) + 4,
                P<long long>(h->arena_off), P<char>(h->arena)};
}

// a table of `slots` slots (a power of two), the entries of the current one re-inserted
int table_resize(c2v_pred* h, unsigned long long slots, cudaStream_t s, const char* fn) {
  Buf key, val;
  PCHECK(fn, cudaMalloc(&key.p, slots * 8));
  key.bytes = slots * 8;
  const cudaError_t e = cudaMalloc(&val.p, slots * 8);
  if (e != cudaSuccess) {
    cudaFree(key.p);
    return pcuda(fn, e);
  }
  val.bytes = slots * 8;
  h->held += 2 * slots * 8;
  if (h->held > h->peak) h->peak = h->held;
  PCHECK(fn, cudaMemsetAsync(key.p, 0, slots * 8, s));
  PCHECK(fn, cudaMemsetAsync(val.p, 0, slots * 8, s));
  PCHECK(fn, cudaMemsetAsync(P<unsigned long long>(h->scalars) + 4, 0, 8, s));
  const unsigned long long old = h->key.p ? h->mask + 1 : 0;
  Unhash nu = table_of(h);
  nu.key = P<unsigned long long>(key);
  nu.val = P<unsigned long long>(val);
  nu.mask = slots - 1;
  if (old) rehash_kernel<<<grid_of((long long)old), kThreads, 0, s>>>(P<unsigned long long>(h->key), P<unsigned long long>(h->val), old, nu);
  PCHECK(fn, cudaGetLastError());
  PCHECK(fn, cudaStreamSynchronize(s));
  for (Buf* b : {&h->key, &h->val})
    if (b->p) {
      cudaFree(b->p);
      h->held -= b->bytes;
    }
  h->key = key;
  h->val = val;
  h->mask = slots - 1;
  return C2V_OK;
}

}  // namespace

int c2v_pred_reset_keys(c2v_pred* h, void* stream) {
  static const char* fn = "c2v_pred_reset_keys";
  if (!h) return pfail(C2V_ERR_INVALID, "c2v_pred_reset_keys: NULL handle");
  PCHECK(fn, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  if ((rc = grow(h, h->scalars, 64, fn))) return rc;
  h->sealed = false;
  if (!h->key.p) return table_resize(h, 1024, s, fn);
  PCHECK(fn, cudaMemsetAsync(h->key.p, 0, h->key.bytes, s));
  PCHECK(fn, cudaMemsetAsync(h->val.p, 0, h->val.bytes, s));
  PCHECK(fn, cudaMemsetAsync(P<unsigned long long>(h->scalars) + 4, 0, 8, s));
  PCHECK(fn, cudaStreamSynchronize(s));
  return C2V_OK;
}

int c2v_pred_seal_keys(c2v_pred* h, void* stream) {
  static const char* fn = "c2v_pred_seal_keys";
  if (!h || !h->key.p) return pfail(C2V_ERR_STATE, "c2v_pred_seal_keys: call c2v_pred_reset_keys first");
  PCHECK(fn, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned long long slots = h->mask + 1;
  int rc;
  if ((rc = grow(h, h->arena_off, slots * 8, fn))) return rc;
  long long* off = P<long long>(h->arena_off);
  arena_len_kernel<<<grid_of((long long)slots), kThreads, 0, s>>>(P<unsigned long long>(h->key), P<unsigned long long>(h->val),
                                                                   slots, off);
  PCHECK(fn, cudaGetLastError());
  long long last_len = 0, last_off = 0;
  PCHECK(fn, cudaMemcpyAsync(&last_len, off + slots - 1, 8, cudaMemcpyDeviceToHost, s));
  size_t tb = 0;
  PCHECK(fn, cub::DeviceScan::ExclusiveSum(nullptr, tb, off, off, (long long)slots, s));
  if ((rc = grow(h, h->tmp, tb, fn))) return rc;
  tb = h->tmp.bytes;
  PCHECK(fn, cub::DeviceScan::ExclusiveSum(h->tmp.p, tb, off, off, (long long)slots, s));
  PCHECK(fn, cudaMemcpyAsync(&last_off, off + slots - 1, 8, cudaMemcpyDeviceToHost, s));
  PCHECK(fn, cudaStreamSynchronize(s));
  if ((rc = grow(h, h->arena, (size_t)(last_off + last_len) + 1, fn))) return rc;
  h->sealed = true;
  return C2V_OK;
}

int c2v_pred_chunk(c2v_pred* h, const char* text, int64_t nbytes, int64_t file_offset, int32_t universal_newlines,
                   int32_t mode, int64_t* n_lines, void* stream) {
  static const char* fn = "c2v_pred_chunk";
  if (!h || !n_lines || nbytes < 0 || file_offset < 0 || (nbytes && !text) || mode < 0 || mode > 2)
    return pfail(C2V_ERR_INVALID, "c2v_pred_chunk: NULL argument, negative size or offset, or mode not in 0..2");
  if (mode != C2V_PRED_SCAN && !h->key.p) return pfail(C2V_ERR_STATE, "c2v_pred_chunk: call c2v_pred_reset_keys first");
  if (mode == C2V_PRED_KEYS && h->sealed) return pfail(C2V_ERR_STATE, "c2v_pred_chunk: the keys are sealed; reset them first");
  if (mode == C2V_PRED_PATHS && !h->sealed) return pfail(C2V_ERR_STATE, "c2v_pred_chunk: seal the keys before copying paths");
  if (mode != C2V_PRED_SCAN && (unsigned long long)(file_offset + nbytes) >= (1ull << (64 - kLenBits)))
    return pfail(C2V_ERR_INVALID, "c2v_pred_chunk: file offsets must stay below 2^44");
  PCHECK(fn, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  const long long n = nbytes;
  int rc;
  if ((rc = grow(h, h->text, (size_t)n + 1, fn)) || (rc = grow(h, h->scalars, 64, fn))) return rc;
  h->n_text = n;
  h->n_lines = 0;
  h->n_rows = 0;
  *n_lines = 0;
  if (n == 0) return C2V_OK;
  PCHECK(fn, cudaMemcpyAsync(h->text.p, text, (size_t)n, cudaMemcpyHostToDevice, s));
  if (mode == C2V_PRED_PATHS) {
    const unsigned long long slots = h->mask + 1;
    arena_copy_kernel<<<grid_of((long long)slots), kThreads, 0, s>>>(P<unsigned char>(h->text), file_offset, n,
                                                                      P<unsigned long long>(h->key),
                                                                      P<unsigned long long>(h->val), slots,
                                                                      P<long long>(h->arena_off), P<char>(h->arena));
    PCHECK(fn, cudaGetLastError());
    PCHECK(fn, cudaStreamSynchronize(s));       // the caller may reuse `text`
    return C2V_OK;
  }
  long long* n_ends_d = P<long long>(h->scalars);
  const IsLineEnd pred{P<unsigned char>(h->text), n, universal_newlines};
  size_t tb = 0;
  {   // count the line ends first: the index then takes 8 bytes per line, not per byte
    const auto ones = thrust::make_transform_iterator(thrust::counting_iterator<long long>(0), LineEndCount{pred});
    PCHECK(fn, cub::DeviceReduce::Sum(nullptr, tb, ones, n_ends_d, n, s));
    if ((rc = grow(h, h->tmp, tb, fn))) return rc;
    tb = h->tmp.bytes;
    PCHECK(fn, cub::DeviceReduce::Sum(h->tmp.p, tb, ones, n_ends_d, n, s));
    long long count = 0;
    PCHECK(fn, cudaMemcpyAsync(&count, n_ends_d, 8, cudaMemcpyDeviceToHost, s));
    PCHECK(fn, cudaStreamSynchronize(s));
    if ((rc = grow(h, h->ends, (size_t)count * 8 + 8, fn))) return rc;
    tb = 0;
  }
  PCHECK(fn, cub::DeviceSelect::If(nullptr, tb, thrust::counting_iterator<long long>(0), P<long long>(h->ends), n_ends_d,
                                   n, pred, s));
  if ((rc = grow(h, h->tmp, tb, fn))) return rc;
  tb = h->tmp.bytes;
  PCHECK(fn, cub::DeviceSelect::If(h->tmp.p, tb, thrust::counting_iterator<long long>(0), P<long long>(h->ends), n_ends_d,
                                   n, pred, s));
  long long n_ends = 0, last_end = -1;
  PCHECK(fn, cudaMemcpyAsync(&n_ends, n_ends_d, 8, cudaMemcpyDeviceToHost, s));
  PCHECK(fn, cudaStreamSynchronize(s));
  if (n_ends) PCHECK(fn, cudaMemcpy(&last_end, P<long long>(h->ends) + n_ends - 1, 8, cudaMemcpyDeviceToHost));
  const long long L = n_ends + (last_end != n - 1 ? 1 : 0);      // text after the last line end is a last line
  if ((rc = grow(h, h->lo, (size_t)L * 8, fn)) || (rc = grow(h, h->hi, (size_t)L * 8, fn)) ||
      (rc = grow(h, h->kind, (size_t)L * 4, fn)) || (rc = grow(h, h->kept, (size_t)L * 4, fn)))
    return rc;
  LineArgs a{P<unsigned char>(h->text), n, P<long long>(h->ends), n_ends, L, h->C, P<long long>(h->lo), P<long long>(h->hi),
             P<int32_t>(h->kind), P<int32_t>(h->kept), table_of(h), 0, file_offset};
  lines_kernel<<<grid_of(L), kThreads, 0, s>>>(a);
  PCHECK(fn, cudaGetLastError());
  if (mode == C2V_PRED_KEYS) {
    // the table keeps at most half its slots in use: grow it for this chunk's kept contexts first
    long long kept = 0;
    unsigned long long used = 0;
    size_t sb = 0;
    long long* sum_d = P<long long>(h->scalars) + 2;
    PCHECK(fn, cub::DeviceReduce::Sum(nullptr, sb, P<int32_t>(h->kept), sum_d, (int)L, s));
    if ((rc = grow(h, h->tmp, sb, fn))) return rc;
    sb = h->tmp.bytes;
    PCHECK(fn, cub::DeviceReduce::Sum(h->tmp.p, sb, P<int32_t>(h->kept), sum_d, (int)L, s));
    PCHECK(fn, cudaMemcpyAsync(&kept, sum_d, 8, cudaMemcpyDeviceToHost, s));
    PCHECK(fn, cudaMemcpyAsync(&used, P<unsigned long long>(h->scalars) + 4, 8, cudaMemcpyDeviceToHost, s));
    PCHECK(fn, cudaStreamSynchronize(s));
    unsigned long long slots = h->mask + 1;
    while (slots < 2ull * (used + (unsigned long long)kept)) slots <<= 1;
    if (slots != h->mask + 1 && (rc = table_resize(h, slots, s, fn))) return rc;
    a.u = table_of(h);
    a.insert = 1;
    lines_kernel<<<grid_of(L), kThreads, 0, s>>>(a);
    PCHECK(fn, cudaGetLastError());
  }
  PCHECK(fn, cudaStreamSynchronize(s));
  h->n_lines = L;
  *n_lines = L;
  return C2V_OK;
}

int c2v_pred_line_info(c2v_pred* h, int64_t* lo, int64_t* hi, int32_t* kind, int32_t* kept) {
  static const char* fn = "c2v_pred_line_info";
  if (!h || !lo || !hi || !kind || !kept) return pfail(C2V_ERR_INVALID, "c2v_pred_line_info: NULL argument");
  if (!h->n_lines) return C2V_OK;
  PCHECK(fn, cudaSetDevice(h->device));
  const size_t L = (size_t)h->n_lines;
  PCHECK(fn, cudaMemcpy(lo, h->lo.p, L * 8, cudaMemcpyDeviceToHost));
  PCHECK(fn, cudaMemcpy(hi, h->hi.p, L * 8, cudaMemcpyDeviceToHost));
  PCHECK(fn, cudaMemcpy(kind, h->kind.p, L * 4, cudaMemcpyDeviceToHost));
  PCHECK(fn, cudaMemcpy(kept, h->kept.p, L * 4, cudaMemcpyDeviceToHost));
  return C2V_OK;
}

int c2v_pred_rows(c2v_pred* h, const int64_t* lines, int32_t n, int32_t* src, int32_t* path, int32_t* tgt, float* mask,
                  void* stream) {
  static const char* fn = "c2v_pred_rows";
  if (!h || !lines || n < 1 || !src || !path || !tgt || !mask) return pfail(C2V_ERR_INVALID, "c2v_pred_rows: NULL argument or n < 1");
  for (int32_t r = 0; r < n; ++r)
    if (lines[r] < 0 || lines[r] >= h->n_lines) return pfail(C2V_ERR_INVALID, "c2v_pred_rows: line number out of range");
  PCHECK(fn, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  const size_t nc = (size_t)n * h->C;
  int rc;
  if ((rc = grow(h, h->line, (size_t)n * 8, fn)) || (rc = grow(h, h->slots, nc * sizeof(Slot), fn)) ||
      (rc = grow(h, h->name, (size_t)n * 16, fn)) || (rc = grow(h, h->code, nc * 4, fn)) || (rc = grow(h, h->fp, nc * 8, fn)))
    return rc;
  PCHECK(fn, cudaMemcpyAsync(h->line.p, lines, (size_t)n * 8, cudaMemcpyHostToDevice, s));
  const RowsArgs a{P<unsigned char>(h->text), P<long long>(h->line), P<long long>(h->lo), P<long long>(h->hi), n, h->C,
                   P<Slot>(h->slots), P<long long>(h->name), h->tok, h->path, src, path, tgt, mask, P<int32_t>(h->code),
                   P<unsigned long long>(h->fp)};
  split_kernel<<<grid_of(n), kThreads, 0, s>>>(a);
  lookup_kernel<<<grid_of((long long)nc), kThreads, 0, s>>>(a);
  PCHECK(fn, cudaGetLastError());
  // the copy of `lines` must not outlive the caller's buffer
  PCHECK(fn, cudaStreamSynchronize(s));
  h->n_rows = n;
  return C2V_OK;
}

int c2v_pred_format(c2v_pred* h, int32_t n, const int32_t* idx, const float* val, int32_t k, const float* attn,
                    const float* code_vec, int32_t code_dim, char* out, int64_t out_cap, int64_t* total, int32_t* bad_row,
                    void* stream) {
  static const char* fn = "c2v_pred_format";
  if (!h || !idx || !val || !attn || !out || !total || !bad_row || k < 1 || (code_vec && code_dim < 1))
    return pfail(C2V_ERR_INVALID, "c2v_pred_format: NULL argument or bad size");
  if (n != h->n_rows || !h->n_words || !h->sealed)
    return pfail(C2V_ERR_STATE, "c2v_pred_format: n must be the rows of the last c2v_pred_rows, after c2v_pred_set_targets "
                                "and c2v_pred_seal_keys");
  PCHECK(fn, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  if ((rc = grow(h, h->top, (size_t)n * kTopContexts * 4, fn)) || (rc = grow(h, h->top_val, (size_t)n * kTopContexts * 4, fn)) ||
      (rc = grow(h, h->row_end, (size_t)n * 8, fn)))
    return rc;
  int32_t* bad_d = P<int32_t>(h->scalars) + 12;
  PCHECK(fn, cudaMemsetAsync(bad_d, 0x7f, 4, s));
  const RankArgs ra{P<unsigned char>(h->text), n, h->C, P<Slot>(h->slots), P<int32_t>(h->code),
                    P<unsigned long long>(h->fp), attn, P<int32_t>(h->top), P<float>(h->top_val), bad_d};
  rank_kernel<<<n, kThreads, (size_t)h->C * 5, s>>>(ra);
  PCHECK(fn, cudaGetLastError());
  const FormatArgs fa{P<unsigned char>(h->text), n, h->C, k, code_dim, P<long long>(h->name), P<Slot>(h->slots),
                      P<int32_t>(h->code), P<int32_t>(h->top), P<float>(h->top_val), idx, val, code_vec,
                      P<char>(h->repr), P<long long>(h->repr_off), h->n_words, h->oov,
                      table_of(h), P<long long>(h->row_end),
                      out, out_cap, bad_d};
  block_len_kernel<<<grid_of(n), kThreads, 0, s>>>(fa);
  size_t tb = 0;
  PCHECK(fn, cub::DeviceScan::InclusiveSum(nullptr, tb, P<long long>(h->row_end), P<long long>(h->row_end), n, s));
  if ((rc = grow(h, h->tmp, tb, fn))) return rc;
  tb = h->tmp.bytes;
  PCHECK(fn, cub::DeviceScan::InclusiveSum(h->tmp.p, tb, P<long long>(h->row_end), P<long long>(h->row_end), n, s));
  block_write_kernel<<<grid_of(n), kThreads, 0, s>>>(fa);
  PCHECK(fn, cudaGetLastError());
  PCHECK(fn, cudaMemcpyAsync(total, P<long long>(h->row_end) + n - 1, 8, cudaMemcpyDeviceToHost, s));
  PCHECK(fn, cudaMemcpyAsync(bad_row, bad_d, 4, cudaMemcpyDeviceToHost, s));
  return C2V_OK;
}

int c2v_selftest_format_fixed(const float* x, int64_t n, char* out, int32_t* len) {
  if (n < 0 || (n && (!x || !out || !len)))
    return pfail(C2V_ERR_INVALID, "c2v_selftest_format_fixed: NULL argument or negative count");
  for (int64_t i = 0; i < n; ++i) {
    char* o = out + i * C2V_FIXED_BYTES;
    len[i] = format_fixed6(x[i], o);
    for (int j = len[i]; j < C2V_FIXED_BYTES; ++j) o[j] = 0;
  }
  return C2V_OK;
}
