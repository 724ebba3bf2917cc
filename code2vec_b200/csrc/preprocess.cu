// Dataset preparation on the device (include/c2v_b200.h "Preprocessing", DESIGN.md §6g): raw extractor output in device
// memory -> the histograms and the down-sampled `.c2v` lines that preprocess.py's count_histograms and process_file
// write, byte for byte.  The text of a chunk is whole lines under universal newlines ('\n', "\r\n" or a lone '\r').
//   utf8       : every byte checked as Python's strict UTF-8 decoder checks it; the lowest bad offset is reported
//   line index : line starts selected from the byte positions (cub::DeviceSelect), one warp per line finds its end,
//                counts its contexts (spaces) and its target's length
//   count      : one warp per line inserts the target and each context's token / path / token parts into one open-
//                addressing table keyed by FNV-1a 64 of (kind, bytes), bytes compared on equal hashes; a new key's bytes
//                go to an arena; per key an atomicAdd count and an atomicMin of the key's first byte offset in the file.
//                The table doubles by rehash before a chunk whose inserts could take it past half full.
//   histogram  : one kind's keys sorted by first offset (Counter insertion order) and printed as `word count\n`
//   classify   : one warp per line records each context's bytes and, on a line of more than max_contexts contexts,
//                probes the two membership tables: full / partial / dropped, and the full-then-partial order
//   assemble   : one warp per output line writes the target, the chosen contexts (the host's picks, or the line as it
//                is), the padding spaces and '\n' at the prefix-summed offset of the line
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <string>

#include "../../include/c2v_b200.h"

namespace c2v {
void set_global_error(const std::string& msg);     // engine.cu: the message c2v_last_error(NULL) returns
}

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kWarps = 8;                          // warps per block of the per-line kernels
constexpr int kBlocks = 132 * 8;                   // grid of the per-line kernels (grid-stride over lines)
constexpr long long kNone = 0x7fffffffffffffffll;

struct DevVocab {                                  // c2v_reader_vocab: native/batcher.cpp Vocab, on the device
  const unsigned long long* slots;                 // 3 words a slot: h, off, (len | idx << 32)
  const unsigned char* bytes;
  unsigned long long mask;
  int32_t oov;
};

struct HSlot {                                     // one histogram key
  unsigned long long h;
  long long off;                                   // its bytes in the arena
  int32_t len, kind;
  unsigned long long count, first;                 // occurrences; the file offset of the first one
  int32_t state, pad;                              // 0 empty, 1 being written, 2 ready
};

struct Counters {                                  // per chunk (reset by reset_kernel) and per table
  long long bad_utf8, lines, inserts, bad_line, seen, kept, written, empty, longest, long_lines;
  long long keys, arena_used;
};

__device__ __forceinline__ unsigned long long fnv1a(const unsigned char* p, long long n, unsigned long long h) {
  for (long long i = 0; i < n; ++i) { h ^= p[i]; h *= 1099511628211ull; }
  return h;
}
constexpr unsigned long long kFnvBasis = 1469598103934665603ull;

// batcher.cpp Vocab::lookup: linear probing from h & mask, the slot with the same hash, length and bytes
__device__ bool member(const DevVocab& v, const unsigned char* p, long long n) {
  unsigned long long h = fnv1a(p, n, kFnvBasis);
  h = h ? h : 1;
  for (unsigned long long i = h & v.mask;; i = (i + 1) & v.mask) {
    const unsigned long long* s = v.slots + 3 * i;
    const unsigned long long sh = s[0];
    if (sh == 0) return false;
    const long long len = (long long)(int32_t)(s[2] & 0xffffffffu);
    if (sh == h && len == n) {
      const unsigned char* w = v.bytes + s[1];
      long long k = 0;
      while (k < n && w[k] == p[k]) ++k;
      if (k == n) return (int32_t)(s[2] >> 32) != v.oov;
    }
  }
}

// ---- UTF-8 ----------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int seq_len(unsigned b) {
  return b < 0x80 ? 1 : b < 0xc2 ? 0 : b < 0xe0 ? 2 : b < 0xf0 ? 3 : b < 0xf5 ? 4 : 0;
}

// Python's strict decoder: no overlong forms (C0, C1, E0 80-9F, F0 80-8F), no surrogates (ED A0-BF), nothing past
// U+10FFFF (F4 90-BF, F5-FF); a byte is bad when it starts no valid sequence and continues none
__global__ void __launch_bounds__(256) utf8_kernel(const unsigned char* __restrict__ t, long long n, Counters* ctr) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const unsigned b = t[i];
    if (b < 0x80) continue;
    bool bad = false;
    if (b < 0xc0) {                                // a continuation byte: covered by the nearest lead before it?
      long long j = i - 1;
      while (j >= 0 && j > i - 4 && t[j] >= 0x80 && t[j] < 0xc0) --j;
      bad = j < 0 || j <= i - 4 || i - j >= seq_len(t[j]);
    } else {
      const int L = seq_len(b);
      bad = L == 0 || i + L > n;
      for (int k = 1; !bad && k < L; ++k) {
        const unsigned c = t[i + k];
        unsigned lo = 0x80, hi = 0xbf;
        if (k == 1) {
          if (b == 0xe0) lo = 0xa0;
          if (b == 0xed) hi = 0x9f;
          if (b == 0xf0) lo = 0x90;
          if (b == 0xf4) hi = 0x8f;
        }
        bad = c < lo || c > hi;
      }
    }
    if (bad) atomicMin(&ctr->bad_utf8, i);
  }
}

// ---- line index -----------------------------------------------------------------------------------------------------
// a line starts at p when p == 0, or after '\n', or after a '\r' that is not followed by '\n' (universal newlines)
struct IsLineStart {
  const unsigned char* t;
  __device__ bool operator()(long long p) const {
    if (p == 0) return true;
    const unsigned char a = t[p - 1];
    return a == '\n' || (a == '\r' && t[p] != '\n');
  }
};

__global__ void reset_kernel(Counters* c) {
  c->bad_utf8 = c->bad_line = kNone;
  c->lines = c->inserts = c->seen = c->kept = c->written = c->empty = c->longest = c->long_lines = 0;
}

// per line: its content's end (the terminator stripped), its contexts (spaces), its target's length; n_ctx[lines] = 0
// closes the array for the scan.  Sums the histogram inserts' bound (1 + spaces + commas a line).
__global__ void __launch_bounds__(kWarps * 32)
line_kernel(const unsigned char* __restrict__ t, long long n, const long long* __restrict__ start,
            const long long* __restrict__ n_lines, long long* __restrict__ end, int32_t* __restrict__ n_ctx,
            int32_t* __restrict__ t_len, Counters* ctr) {
  __shared__ unsigned long long s_ins;
  if (threadIdx.x == 0) s_ins = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long L = *n_lines;
  unsigned long long ins = 0;
  for (long long l = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; l < L; l += ((long long)gridDim.x * blockDim.x) >> 5) {
    const long long s = start[l];
    long long e = l + 1 < L ? start[l + 1] : n;
    while (e > s && (t[e - 1] == '\n' || t[e - 1] == '\r')) --e;
    long long spaces = 0, commas = 0, first = -1;
    for (long long w = s; w < e; w += 32) {
      const long long p = w + lane;
      const unsigned char c = p < e ? t[p] : 0;
      const unsigned sp = __ballot_sync(kFull, c == ' '), cm = __ballot_sync(kFull, c == ',');
      if (first < 0 && sp) first = w + __ffs(sp) - 1 - s;
      spaces += __popc(sp);
      commas += __popc(cm);
    }
    if (lane == 0) {
      end[l] = e;
      n_ctx[l] = (int32_t)spaces;
      t_len[l] = (int32_t)(first < 0 ? e - s : first);
      ins += 1 + spaces + commas;
    }
  }
  if (lane == 0 && ins) atomicAdd(&s_ins, ins);
  __syncthreads();
  if (threadIdx.x == 0) {
    atomicAdd((unsigned long long*)&ctr->inserts, s_ins);
    if (blockIdx.x == 0) { n_ctx[L] = 0; ctr->lines = L; }
  }
}

// The fields of line [s, e): f(index, a, b) for every space-separated field [a, b), field 0 being the target.  Each
// field is handled by the lane that holds the space after it (the line's last field by lane 0).
template <typename F>
__device__ __forceinline__ void for_each_field(const unsigned char* t, long long s, long long e, int lane, F&& f) {
  const unsigned lt = (1u << lane) - 1;
  long long nf = 0, last = s - 1;
  for (long long w = s; w < e; w += 32) {
    const long long p = w + lane;
    const unsigned char c = p < e ? t[p] : 0;
    const unsigned sp = __ballot_sync(kFull, c == ' ');
    if (c == ' ') {
      const unsigned before = sp & lt;
      const long long a = before ? w + (31 - __clz(before)) + 1 : last + 1;
      f(nf + __popc(before), a, p);
    }
    if (sp) last = w + (31 - __clz(sp));
    nf += __popc(sp);
  }
  if (lane == 0) f(nf, last + 1, e);
}

// the first comma in [a, b), or b
__device__ __forceinline__ long long comma(const unsigned char* t, long long a, long long b) {
  while (a < b && t[a] != ',') ++a;
  return a;
}

// ---- histogram table ------------------------------------------------------------------------------------------------
struct Table {
  HSlot* slots;
  unsigned long long mask;
  unsigned char* arena;
  Counters* ctr;
};

__device__ __forceinline__ unsigned long long key_hash(int kind, const unsigned char* p, long long n) {
  unsigned long long h = fnv1a(p, n, (kFnvBasis ^ (unsigned long long)kind) * 1099511628211ull);
  return h ? h : 1;
}

__device__ __forceinline__ void wait_ready(const HSlot* s) {
  while (*(volatile const int32_t*)&s->state != 2) __nanosleep(20);
  __threadfence();
}

__device__ void insert(const Table& tb, int kind, const unsigned char* p, long long n, unsigned long long off) {
  const unsigned long long h = key_hash(kind, p, n);
  for (unsigned long long i = h & tb.mask;; i = (i + 1) & tb.mask) {
    HSlot* s = tb.slots + i;
    int32_t st = *(volatile int32_t*)&s->state;
    if (st == 0) {
      st = atomicCAS(&s->state, 0, 1);
      if (st == 0) {                               // claimed: copy the key's bytes to the arena, then publish the slot
        const long long a = (long long)atomicAdd((unsigned long long*)&tb.ctr->arena_used, (unsigned long long)n);
        for (long long k = 0; k < n; ++k) tb.arena[a + k] = p[k];
        s->h = h;
        s->off = a;
        s->len = (int32_t)n;
        s->kind = kind;
        s->count = 1;
        s->first = off;
        atomicAdd((unsigned long long*)&tb.ctr->keys, 1ull);
        __threadfence();
        atomicExch(&s->state, 2);
        return;
      }
    }
    wait_ready(s);
    if (s->h == h && s->kind == kind && (long long)s->len == n) {
      const unsigned char* w = tb.arena + s->off;
      long long k = 0;
      while (k < n && w[k] == p[k]) ++k;
      if (k == n) {
        atomicAdd(&s->count, 1ull);
        atomicMin(&s->first, off);
        return;
      }
    }
  }
}

// count_histograms for one chunk: target, then per context tokens[p0], paths[p1], tokens[p2] (three parts or more) or
// tokens[p0] and paths[p1] if there is a second part
__global__ void __launch_bounds__(kWarps * 32)
count_kernel(const unsigned char* __restrict__ t, const long long* __restrict__ start, const long long* __restrict__ end,
             const long long* __restrict__ n_lines, unsigned long long base, Table tb) {
  const int lane = threadIdx.x & 31;
  const long long L = *n_lines;
  for (long long l = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; l < L; l += ((long long)gridDim.x * blockDim.x) >> 5) {
    for_each_field(t, start[l], end[l], lane, [&](long long f, long long a, long long b) {
      if (f == 0) {
        insert(tb, 2, t + a, b - a, base + a);
        return;
      }
      const long long c1 = comma(t, a, b);
      insert(tb, 0, t + a, c1 - a, base + a);
      if (c1 == b) return;
      const long long c2 = comma(t, c1 + 1, b);
      insert(tb, 1, t + c1 + 1, c2 - c1 - 1, base + c1 + 1);
      if (c2 == b) return;
      const long long c3 = comma(t, c2 + 1, b);
      insert(tb, 0, t + c2 + 1, c3 - c2 - 1, base + c2 + 1);
    });
    __syncwarp();
  }
}

// every ready slot of the old table into the new one (keys are distinct: no comparison)
__global__ void __launch_bounds__(256) rehash_kernel(const HSlot* __restrict__ old, unsigned long long old_slots, HSlot* nw,
                                                     unsigned long long mask) {
  for (unsigned long long i = (unsigned long long)blockIdx.x * 256 + threadIdx.x; i < old_slots;
       i += (unsigned long long)gridDim.x * 256) {
    const HSlot s = old[i];
    if (s.state != 2) continue;
    for (unsigned long long j = s.h & mask;; j = (j + 1) & mask) {
      if (atomicCAS(&nw[j].state, 0, 1) == 0) {
        nw[j] = s;
        break;
      }
    }
  }
}

struct IsKind {
  const HSlot* slots;
  int kind;
  __device__ bool operator()(long long i) const { return slots[i].state == 2 && slots[i].kind == kind; }
};

__device__ __forceinline__ int digits(unsigned long long v) {
  int d = 1;
  while (v >= 10) { v /= 10; ++d; }
  return d;
}

__global__ void __launch_bounds__(256) first_kernel(const HSlot* __restrict__ slots, const long long* __restrict__ idx,
                                                    const long long* __restrict__ n, unsigned long long* __restrict__ key) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < *n; i += (long long)gridDim.x * 256)
    key[i] = slots[idx[i]].first;
}

// len[i] = the bytes of `word count\n` for key i (sorted order); len[n] = 0 closes the array for the scan
__global__ void __launch_bounds__(256) histo_len_kernel(const HSlot* __restrict__ slots, const long long* __restrict__ idx,
                                                        const long long* __restrict__ n, long long* __restrict__ len) {
  const long long N = *n;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i <= N; i += (long long)gridDim.x * 256) {
    if (i == N) { len[i] = 0; continue; }
    const HSlot& s = slots[idx[i]];
    len[i] = s.len + 2 + digits(s.count);
  }
}

__global__ void __launch_bounds__(256) histo_write_kernel(const HSlot* __restrict__ slots, const unsigned char* __restrict__ arena,
                                                          const long long* __restrict__ idx, const long long* __restrict__ n,
                                                          const long long* __restrict__ off, char* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < *n; i += (long long)gridDim.x * 256) {
    const HSlot& s = slots[idx[i]];
    char* o = out + off[i];
    for (int k = 0; k < s.len; ++k) o[k] = (char)arena[s.off + k];
    o += s.len;
    *o++ = ' ';
    const int d = digits(s.count);
    unsigned long long v = s.count;
    for (int k = d - 1; k >= 0; --k) { o[k] = (char)('0' + v % 10); v /= 10; }
    o[d] = '\n';
  }
}

// ---- classify and assemble ------------------------------------------------------------------------------------------
struct Lines {
  const unsigned char* t;
  const long long *start, *end, *n_lines;
  const int32_t *n_ctx, *t_len;
  const int32_t* ctx_base;                         // exclusive scan of n_ctx: a line's first context
  int32_t *ctx_start, *ctx_len;                    // per context: offset in the chunk, bytes
  int8_t* cls;                                     // per context of a long line: 2 full, 1 partial, 0 dropped
  int32_t* order;                                  // per long line: its full contexts, then its partial ones
  int32_t *n_full, *n_part, *kept;
  int C;
};

__global__ void __launch_bounds__(kWarps * 32) classify_kernel(Lines a, DevVocab tok, DevVocab pth, Counters* ctr) {
  __shared__ unsigned long long s_sum[4];          // seen, kept, written, empty
  __shared__ long long s_longest, s_bad;
  if (threadIdx.x < 4) s_sum[threadIdx.x] = 0;
  if (threadIdx.x == 0) { s_longest = 0; s_bad = kNone; }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1;
  const long long L = *a.n_lines;
  const int C = a.C;
  for (long long l = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; l < L; l += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int n = a.n_ctx[l];
    const int base = a.ctx_base[l];
    const bool is_long = n > C;
    bool short_part = false;
    for_each_field(a.t, a.start[l], a.end[l], lane, [&](long long f, long long x, long long y) {
      if (f == 0) return;
      const int j = base + (int)f - 1;
      a.ctx_start[j] = (int32_t)x;
      a.ctx_len[j] = (int32_t)(y - x);
      if (!is_long) return;
      const long long c1 = comma(a.t, x, y);
      const long long c2 = c1 < y ? comma(a.t, c1 + 1, y) : y;
      if (c2 >= y) {                               // fewer than three parts: parts[1] or parts[2] raises IndexError
        short_part = true;
        a.cls[j] = 0;
        return;
      }
      const long long c3 = comma(a.t, c2 + 1, y);
      const bool k0 = member(tok, a.t + x, c1 - x), k1 = member(pth, a.t + c1 + 1, c2 - c1 - 1),
                 k2 = member(tok, a.t + c2 + 1, c3 - c2 - 1);
      a.cls[j] = (k0 && k1 && k2) ? 2 : (k0 || k1 || k2) ? 1 : 0;
    });
    __syncwarp();
    int nf = 0, np = 0;
    if (is_long) {
      for (int j0 = 0; j0 < n; j0 += 32) {
        const int c = j0 + lane < n ? a.cls[base + j0 + lane] : 0;
        nf += __popc(__ballot_sync(kFull, c == 2));
        np += __popc(__ballot_sync(kFull, c == 1));
      }
      int rf = 0, rp = nf;
      for (int j0 = 0; j0 < n; j0 += 32) {
        const int c = j0 + lane < n ? a.cls[base + j0 + lane] : 0;
        const unsigned bf = __ballot_sync(kFull, c == 2), bp = __ballot_sync(kFull, c == 1);
        if (c == 2) a.order[base + rf + __popc(bf & lt)] = j0 + lane;
        if (c == 1) a.order[base + rp + __popc(bp & lt)] = j0 + lane;
        rf += __popc(bf);
        rp += __popc(bp);
      }
    }
    const bool bad = __any_sync(kFull, short_part) && is_long;
    if (lane == 0) {
      const int kept = is_long ? min(C, nf + np) : n;
      a.n_full[l] = nf;
      a.n_part[l] = np;
      a.kept[l] = kept;
      atomicAdd(&s_sum[0], (unsigned long long)n);
      atomicAdd(&s_sum[1], (unsigned long long)kept);
      atomicAdd(&s_sum[kept ? 2 : 3], 1ull);
      atomicMax((unsigned long long*)&s_longest, (unsigned long long)n);
      if (bad) atomicMin(&s_bad, l);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    atomicAdd((unsigned long long*)&ctr->seen, s_sum[0]);
    atomicAdd((unsigned long long*)&ctr->kept, s_sum[1]);
    atomicAdd((unsigned long long*)&ctr->written, s_sum[2]);
    atomicAdd((unsigned long long*)&ctr->empty, s_sum[3]);
    atomicMax(&ctr->longest, s_longest);
    if (s_bad != kNone) atomicMin(&ctr->bad_line, s_bad);
  }
}

struct IsLong {
  const int32_t* n_ctx;
  int C;
  __device__ bool operator()(long long l) const { return n_ctx[l] > C; }
};

// per long line r: long_rank[its line] = r, and its counts for the host
__global__ void __launch_bounds__(256) long_kernel(const long long* __restrict__ idx, const long long* __restrict__ n,
                                                   const int32_t* __restrict__ n_full, const int32_t* __restrict__ n_part,
                                                   int32_t* __restrict__ long_rank, int32_t* __restrict__ nf_out,
                                                   int32_t* __restrict__ np_out, Counters* ctr) {
  const long long N = *n;
  for (long long r = (long long)blockIdx.x * 256 + threadIdx.x; r < N; r += (long long)gridDim.x * 256) {
    const long long l = idx[r];
    long_rank[l] = (int32_t)r;
    nf_out[r] = n_full[l];
    np_out[r] = n_part[l];
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) ctr->long_lines = N;
}

struct Picks {
  const int32_t* long_rank;
  const int32_t* picks;                            // the host's rng.sample(range(m), k) results, long lines in order
  const long long* pick_off;                       // [long lines + 1]
};

// the index (within its line) of output context j of line l
__device__ __forceinline__ int chosen(const Lines& a, const Picks& pk, long long l, int j) {
  const int n = a.n_ctx[l];
  if (n <= a.C) return j;
  const int base = a.ctx_base[l], nf = a.n_full[l], np = a.n_part[l];
  const long long po = pk.pick_off[pk.long_rank[l]];
  if (nf > a.C) return a.order[base + pk.picks[po + j]];
  if (nf + np > a.C) return j < nf ? a.order[base + j] : a.order[base + nf + pk.picks[po + j - nf]];
  return a.order[base + j];
}

// out_len[l] = target + ' ' + the chosen contexts joined by ' ' + the padding + '\n' (0 for a line left empty)
__global__ void __launch_bounds__(kWarps * 32) out_len_kernel(Lines a, Picks pk, long long* __restrict__ out_len) {
  const int lane = threadIdx.x & 31;
  const long long L = *a.n_lines;
  for (long long l = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; l < L; l += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int kept = a.kept[l], base = a.ctx_base[l];
    long long sum = 0;
    for (int j = lane; j < kept; j += 32) sum += a.ctx_len[base + chosen(a, pk, l, j)];
    sum = __reduce_add_sync(kFull, (unsigned)sum);
    if (lane == 0) out_len[l] = kept ? a.t_len[l] + sum + a.C + 1 : 0;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) out_len[L] = 0;
}

__global__ void __launch_bounds__(kWarps * 32) assemble_kernel(Lines a, Picks pk, const long long* __restrict__ out_off,
                                                               char* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long L = *a.n_lines;
  for (long long l = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; l < L; l += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int kept = a.kept[l];
    if (!kept) continue;
    const int base = a.ctx_base[l], tl = a.t_len[l];
    char* o = out + out_off[l];
    const unsigned char* src = a.t + a.start[l];
    for (int k = lane; k < tl; k += 32) o[k] = (char)src[k];
    if (lane == 0) o[tl] = ' ';
    long long pos = tl + 1;
    for (int j0 = 0; j0 < kept; j0 += 32) {
      const int j = j0 + lane;
      int s = 0, n = 0;
      if (j < kept) {
        const int c = base + chosen(a, pk, l, j);
        s = a.ctx_start[c];
        n = a.ctx_len[c] + 1;                      // the context and the space after it
      }
      int incl = n;
      for (int d = 1; d < 32; d <<= 1) {
        const int v = __shfl_up_sync(kFull, incl, d);
        if (lane >= d) incl += v;
      }
      if (j < kept) {
        char* q = o + pos + incl - n;
        for (int k = 0; k < n - 1; ++k) q[k] = (char)a.t[s + k];
        q[n - 1] = ' ';
      }
      pos += __shfl_sync(kFull, incl, 31);
    }
    // pos is one past the last context's space; up to the '\n' at tl + sum + C everything is padding
    const long long nl = out_off[l + 1] - out_off[l] - 1;
    for (long long k = pos + lane; k < nl; k += 32) o[k] = ' ';
    __syncwarp();
    if (lane == 0) o[nl] = '\n';
  }
}

}  // namespace

// ---- the handle -------------------------------------------------------------------------------------------------------
struct c2v_prep {
  int device = 0;
  size_t held = 0;
  Counters* ctr = nullptr;                         // device
  Counters host{};
  // histogram table
  HSlot* slots = nullptr;
  unsigned long long n_slots = 0;
  unsigned char* arena = nullptr;
  size_t arena_cap = 0;
  long long rehashes = 0;
  // per chunk
  const unsigned char* text = nullptr;
  long long nbytes = 0;
  int C = 0;
  bool classified = false;
  struct Buf { void* p = nullptr; size_t cap = 0; };
  Buf temp, start, end, n_ctx, t_len, ctx_base, ctx_start, ctx_len, cls, order, n_full, n_part, kept, long_idx, long_rank,
      long_nf, long_np, picks, pick_off, out_len, out_off, out, hidx, hidx2, hkey, hkey2, n_sel;
};

namespace {

int pfail(int code, const std::string& msg) {
  c2v::set_global_error(msg);
  return code;
}

int cuda_fail(const char* fn, cudaError_t e) { return pfail(C2V_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(e)); }

#define PCHECK(fn, x)                                   \
  do {                                                  \
    const cudaError_t e_ = (x);                         \
    if (e_ != cudaSuccess) return cuda_fail(fn, e_);   \
  } while (0)

cudaError_t grow(c2v_prep* h, c2v_prep::Buf& b, size_t bytes) {
  if (bytes <= b.cap) return cudaSuccess;
  bytes = bytes < 256 ? 256 : bytes + bytes / 4;
  if (b.p) { cudaFree(b.p); h->held -= b.cap; b.p = nullptr; b.cap = 0; }
  const cudaError_t e = cudaMalloc(&b.p, bytes);
  if (e == cudaSuccess) { b.cap = bytes; h->held += bytes; }
  return e;
}

template <typename T> T* P(const c2v_prep::Buf& b) { return (T*)b.p; }

cudaError_t read_counters(c2v_prep* h, cudaStream_t s) {
  cudaError_t e = cudaMemcpyAsync(&h->host, h->ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  return e;
}

// cub's device-wide algorithms with the handle's scratch
template <typename F> cudaError_t with_temp(c2v_prep* h, F&& f) {
  size_t need = 0;
  cudaError_t e = f(nullptr, need);
  if (e == cudaSuccess) e = grow(h, h->temp, need);
  if (e == cudaSuccess) { need = h->temp.cap; e = f(h->temp.p, need); }
  return e;
}

// utf8 check and line index of text[0, nbytes), then the counters read back
int index_chunk(c2v_prep* h, const char* fn, const char* text, int64_t nbytes, cudaStream_t s) {
  if (nbytes < 0 || nbytes >= (1ll << 31) || (nbytes && !text))
    return pfail(C2V_ERR_INVALID, std::string(fn) + ": need 0 <= nbytes < 2^31 and a text pointer");
  h->text = (const unsigned char*)text;
  h->nbytes = nbytes;
  h->classified = false;
  const long long n = nbytes;
  PCHECK(fn, grow(h, h->start, (n + 1) * 8));
  PCHECK(fn, grow(h, h->end, (n + 1) * 8));
  PCHECK(fn, grow(h, h->n_ctx, (n + 2) * 4));
  PCHECK(fn, grow(h, h->t_len, (n + 1) * 4));
  PCHECK(fn, grow(h, h->n_sel, 16));       // [0] lines, [1] long lines
  reset_kernel<<<1, 1, 0, s>>>(h->ctr);
  PCHECK(fn, cudaMemsetAsync(h->n_sel.p, 0, 16, s));
  if (n) {
    utf8_kernel<<<(unsigned)std::min<long long>((n + 255) / 256, 132 * 16), 256, 0, s>>>(h->text, n, h->ctr);
    IsLineStart pred{h->text};
    long long* out = P<long long>(h->start);
    long long* num = P<long long>(h->n_sel);
    PCHECK(fn, with_temp(h, [&](void* tmp, size_t& bytes) {
      return cub::DeviceSelect::If(tmp, bytes, thrust::counting_iterator<long long>(0), out, num, n, pred, s);
    }));
  }
  line_kernel<<<kBlocks, kWarps * 32, 0, s>>>(h->text, n, P<long long>(h->start), P<long long>(h->n_sel),
                                               P<long long>(h->end), P<int32_t>(h->n_ctx), P<int32_t>(h->t_len), h->ctr);
  PCHECK(fn, cudaGetLastError());
  PCHECK(fn, read_counters(h, s));
  return C2V_OK;
}

void fill_status(const c2v_prep* h, c2v_prep_status* st) {
  const Counters& c = h->host;
  st->lines = c.lines;
  st->bad_utf8 = c.bad_utf8 == kNone ? -1 : c.bad_utf8;
  st->bad_line = c.bad_line == kNone ? -1 : c.bad_line;
  st->long_lines = c.long_lines;
  st->seen = c.seen;
  st->kept = c.kept;
  st->written = c.written;
  st->empty = c.empty;
  st->longest = c.longest;
  st->keys = c.keys;
  st->slots = (int64_t)h->n_slots;
  st->rehashes = h->rehashes;
}

Lines lines_of(c2v_prep* h) {
  Lines a;
  a.t = h->text;
  a.start = P<long long>(h->start);
  a.end = P<long long>(h->end);
  a.n_lines = P<long long>(h->n_sel);
  a.n_ctx = P<int32_t>(h->n_ctx);
  a.t_len = P<int32_t>(h->t_len);
  a.ctx_base = P<int32_t>(h->ctx_base);
  a.ctx_start = P<int32_t>(h->ctx_start);
  a.ctx_len = P<int32_t>(h->ctx_len);
  a.cls = P<int8_t>(h->cls);
  a.order = P<int32_t>(h->order);
  a.n_full = P<int32_t>(h->n_full);
  a.n_part = P<int32_t>(h->n_part);
  a.kept = P<int32_t>(h->kept);
  a.C = h->C;
  return a;
}

}  // namespace

int c2v_prep_create(int device, c2v_prep** out) {
  if (!out) return pfail(C2V_ERR_INVALID, "c2v_prep_create: NULL out");
  *out = nullptr;
  PCHECK("c2v_prep_create", cudaSetDevice(device));
  c2v_prep* h = new c2v_prep();
  h->device = device;
  cudaError_t e = cudaMalloc(&h->ctr, sizeof(Counters));
  if (e == cudaSuccess) e = cudaMemset(h->ctr, 0, sizeof(Counters));
  if (e != cudaSuccess) {
    c2v_prep_destroy(h);
    return cuda_fail("c2v_prep_create", e);
  }
  h->held += sizeof(Counters);
  *out = h;
  return C2V_OK;
}

void c2v_prep_destroy(c2v_prep* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  for (c2v_prep::Buf* b : {&h->temp, &h->start, &h->end, &h->n_ctx, &h->t_len, &h->ctx_base, &h->ctx_start, &h->ctx_len,
                           &h->cls, &h->order, &h->n_full, &h->n_part, &h->kept, &h->long_idx, &h->long_rank, &h->long_nf,
                           &h->long_np, &h->picks, &h->pick_off, &h->out_len, &h->out_off, &h->out, &h->hidx, &h->hidx2,
                           &h->hkey, &h->hkey2, &h->n_sel})
    if (b->p) cudaFree(b->p);
  if (h->slots) cudaFree(h->slots);
  if (h->arena) cudaFree(h->arena);
  if (h->ctr) cudaFree(h->ctr);
  delete h;
}

size_t c2v_prep_device_bytes(const c2v_prep* h) {
  return h ? h->held + h->n_slots * sizeof(HSlot) + h->arena_cap : 0;
}

int c2v_prep_count_chunk(c2v_prep* h, const char* text, int64_t nbytes, int64_t file_offset, c2v_prep_status* st,
                         void* stream) {
  const char* fn = "c2v_prep_count_chunk";
  if (!h || !st || file_offset < 0) return pfail(C2V_ERR_INVALID, "c2v_prep_count_chunk: NULL argument or negative offset");
  cudaStream_t s = (cudaStream_t)stream;
  PCHECK(fn, cudaSetDevice(h->device));
  int rc = index_chunk(h, fn, text, nbytes, s);
  if (rc) return rc;
  if (h->host.bad_utf8 != kNone) {
    fill_status(h, st);
    return C2V_OK;
  }
  // room for every insert of the chunk being a new key: at most half full, and the key bytes in the arena
  const unsigned long long need = (unsigned long long)(h->host.keys + h->host.inserts) * 2;
  unsigned long long cap = h->n_slots ? h->n_slots : 1024;
  while (cap < need) cap <<= 1;
  if (cap != h->n_slots) {
    HSlot* nw = nullptr;
    PCHECK(fn, cudaMalloc(&nw, cap * sizeof(HSlot)));
    PCHECK(fn, cudaMemsetAsync(nw, 0, cap * sizeof(HSlot), s));
    if (h->n_slots) {
      rehash_kernel<<<(unsigned)std::min<unsigned long long>((h->n_slots + 255) / 256, 132 * 16), 256, 0, s>>>(
          h->slots, h->n_slots, nw, cap - 1);
      PCHECK(fn, cudaGetLastError());
      if (h->host.keys) ++h->rehashes;
      PCHECK(fn, cudaStreamSynchronize(s));
      cudaFree(h->slots);
    }
    h->slots = nw;
    h->n_slots = cap;
  }
  const size_t arena_need = (size_t)h->host.arena_used + (size_t)nbytes + 1;
  if (arena_need > h->arena_cap) {
    const size_t cap_b = arena_need + arena_need / 2;
    unsigned char* a = nullptr;
    PCHECK(fn, cudaMalloc(&a, cap_b));
    if (h->arena) {
      PCHECK(fn, cudaMemcpyAsync(a, h->arena, (size_t)h->host.arena_used, cudaMemcpyDeviceToDevice, s));
      PCHECK(fn, cudaStreamSynchronize(s));
      cudaFree(h->arena);
    }
    h->arena = a;
    h->arena_cap = cap_b;
  }
  Table tb{h->slots, h->n_slots - 1, h->arena, h->ctr};
  count_kernel<<<kBlocks, kWarps * 32, 0, s>>>(h->text, P<long long>(h->start), P<long long>(h->end),
                                                P<long long>(h->n_sel), (unsigned long long)file_offset, tb);
  PCHECK(fn, cudaGetLastError());
  PCHECK(fn, read_counters(h, s));
  fill_status(h, st);
  return C2V_OK;
}

int c2v_prep_histogram(c2v_prep* h, int32_t kind, const char** text, int64_t* nbytes, void* stream) {
  const char* fn = "c2v_prep_histogram";
  if (!h || !text || !nbytes || kind < 0 || kind > 2)
    return pfail(C2V_ERR_INVALID, "c2v_prep_histogram: NULL argument or kind not in 0..2");
  cudaStream_t s = (cudaStream_t)stream;
  PCHECK(fn, cudaSetDevice(h->device));
  *text = nullptr;
  *nbytes = 0;
  if (!h->n_slots) return C2V_OK;
  const long long cap = (long long)h->n_slots, keys = h->host.keys + 1;     // the kind's keys are among all keys
  PCHECK(fn, grow(h, h->hidx, keys * 8));
  PCHECK(fn, grow(h, h->hidx2, keys * 8));
  PCHECK(fn, grow(h, h->hkey, keys * 8));
  PCHECK(fn, grow(h, h->hkey2, keys * 8));
  PCHECK(fn, grow(h, h->out_len, (keys + 1) * 8));
  PCHECK(fn, grow(h, h->out_off, (keys + 1) * 8));
  long long* idx = P<long long>(h->hidx);
  long long* num = P<long long>(h->n_sel);
  IsKind pred{h->slots, kind};
  PCHECK(fn, with_temp(h, [&](void* tmp, size_t& bytes) {
    return cub::DeviceSelect::If(tmp, bytes, thrust::counting_iterator<long long>(0), idx, num, cap, pred, s);
  }));
  long long n = 0;
  PCHECK(fn, cudaMemcpyAsync(&n, num, 8, cudaMemcpyDeviceToHost, s));
  PCHECK(fn, cudaStreamSynchronize(s));
  if (!n) return C2V_OK;
  const unsigned grid = (unsigned)std::min<long long>((n + 256) / 256, 132 * 16);
  first_kernel<<<grid, 256, 0, s>>>(h->slots, idx, num, P<unsigned long long>(h->hkey));
  PCHECK(fn, cudaGetLastError());
  unsigned long long* k_in = P<unsigned long long>(h->hkey);
  unsigned long long* k_out = P<unsigned long long>(h->hkey2);
  long long* v_out = P<long long>(h->hidx2);
  PCHECK(fn, with_temp(h, [&](void* tmp, size_t& bytes) {
    return cub::DeviceRadixSort::SortPairs(tmp, bytes, k_in, k_out, idx, v_out, (int)n, 0, 64, s);
  }));
  long long* len = P<long long>(h->out_len);
  long long* off = P<long long>(h->out_off);
  histo_len_kernel<<<grid, 256, 0, s>>>(h->slots, v_out, num, len);
  PCHECK(fn, with_temp(h, [&](void* tmp, size_t& bytes) {
    return cub::DeviceScan::ExclusiveSum(tmp, bytes, len, off, (int)(n + 1), s);
  }));
  long long total = 0;
  PCHECK(fn, cudaMemcpyAsync(&total, off + n, 8, cudaMemcpyDeviceToHost, s));
  PCHECK(fn, cudaStreamSynchronize(s));
  PCHECK(fn, grow(h, h->out, (size_t)total));
  histo_write_kernel<<<grid, 256, 0, s>>>(h->slots, h->arena, v_out, num, off, P<char>(h->out));
  PCHECK(fn, cudaGetLastError());
  *text = P<char>(h->out);
  *nbytes = total;
  return C2V_OK;
}

int c2v_prep_classify_chunk(c2v_prep* h, const char* text, int64_t nbytes, int32_t max_contexts,
                            const c2v_reader_vocab* token, const c2v_reader_vocab* path, c2v_prep_status* st,
                            void* stream) {
  const char* fn = "c2v_prep_classify_chunk";
  if (!h || !st || !token || !path || max_contexts < 0)
    return pfail(C2V_ERR_INVALID, "c2v_prep_classify_chunk: NULL argument or negative max_contexts");
  cudaStream_t s = (cudaStream_t)stream;
  PCHECK(fn, cudaSetDevice(h->device));
  int rc = index_chunk(h, fn, text, nbytes, s);
  if (rc) return rc;
  h->C = max_contexts;
  if (h->host.bad_utf8 != kNone) {
    fill_status(h, st);
    return C2V_OK;
  }
  const long long L = h->host.lines;
  PCHECK(fn, grow(h, h->ctx_base, (L + 1) * 4));
  PCHECK(fn, grow(h, h->n_full, (L + 1) * 4));
  PCHECK(fn, grow(h, h->n_part, (L + 1) * 4));
  PCHECK(fn, grow(h, h->kept, (L + 1) * 4));
  PCHECK(fn, grow(h, h->long_rank, (L + 1) * 4));
  PCHECK(fn, grow(h, h->long_idx, (L + 1) * 8));
  PCHECK(fn, grow(h, h->long_nf, (L + 1) * 4));
  PCHECK(fn, grow(h, h->long_np, (L + 1) * 4));
  int32_t* n_ctx = P<int32_t>(h->n_ctx);
  int32_t* base = P<int32_t>(h->ctx_base);
  PCHECK(fn, with_temp(h, [&](void* tmp, size_t& bytes) {
    return cub::DeviceScan::ExclusiveSum(tmp, bytes, n_ctx, base, (int)(L + 1), s);
  }));
  int32_t total = 0;
  PCHECK(fn, cudaMemcpyAsync(&total, base + L, 4, cudaMemcpyDeviceToHost, s));
  PCHECK(fn, cudaStreamSynchronize(s));
  PCHECK(fn, grow(h, h->ctx_start, ((size_t)total + 1) * 4));
  PCHECK(fn, grow(h, h->ctx_len, ((size_t)total + 1) * 4));
  PCHECK(fn, grow(h, h->cls, (size_t)total + 1));
  PCHECK(fn, grow(h, h->order, ((size_t)total + 1) * 4));
  const DevVocab tok{(const unsigned long long*)token->slots, (const unsigned char*)token->bytes, token->mask, token->oov};
  const DevVocab pth{(const unsigned long long*)path->slots, (const unsigned char*)path->bytes, path->mask, path->oov};
  classify_kernel<<<kBlocks, kWarps * 32, 0, s>>>(lines_of(h), tok, pth, h->ctr);
  PCHECK(fn, cudaGetLastError());
  long long* idx = P<long long>(h->long_idx);
  IsLong pred{n_ctx, max_contexts};
  PCHECK(fn, with_temp(h, [&](void* tmp, size_t& bytes) {
    return cub::DeviceSelect::If(tmp, bytes, thrust::counting_iterator<long long>(0), idx, P<long long>(h->n_sel) + 1, L, pred, s);
  }));
  long_kernel<<<kBlocks, 256, 0, s>>>(idx, P<long long>(h->n_sel) + 1, P<int32_t>(h->n_full), P<int32_t>(h->n_part),
                                       P<int32_t>(h->long_rank), P<int32_t>(h->long_nf), P<int32_t>(h->long_np), h->ctr);
  PCHECK(fn, cudaGetLastError());
  PCHECK(fn, read_counters(h, s));
  h->classified = true;
  fill_status(h, st);
  return C2V_OK;
}

int c2v_prep_long_lines(c2v_prep* h, int64_t* line, int32_t* n_full, int32_t* n_partial, void* stream) {
  const char* fn = "c2v_prep_long_lines";
  if (!h || !h->classified) return pfail(C2V_ERR_STATE, "c2v_prep_long_lines: no classified chunk");
  const long long n = h->host.long_lines;
  if (n && (!line || !n_full || !n_partial)) return pfail(C2V_ERR_INVALID, "c2v_prep_long_lines: NULL argument");
  cudaStream_t s = (cudaStream_t)stream;
  PCHECK(fn, cudaSetDevice(h->device));
  if (!n) return C2V_OK;
  PCHECK(fn, cudaMemcpyAsync(line, h->long_idx.p, n * 8, cudaMemcpyDeviceToHost, s));
  PCHECK(fn, cudaMemcpyAsync(n_full, h->long_nf.p, n * 4, cudaMemcpyDeviceToHost, s));
  PCHECK(fn, cudaMemcpyAsync(n_partial, h->long_np.p, n * 4, cudaMemcpyDeviceToHost, s));
  PCHECK(fn, cudaStreamSynchronize(s));
  return C2V_OK;
}

int c2v_prep_assemble(c2v_prep* h, const int32_t* picks, const int64_t* pick_off, const char** text, int64_t* nbytes,
                      void* stream) {
  const char* fn = "c2v_prep_assemble";
  if (!h || !h->classified) return pfail(C2V_ERR_STATE, "c2v_prep_assemble: no classified chunk");
  if (!text || !nbytes || !pick_off) return pfail(C2V_ERR_INVALID, "c2v_prep_assemble: NULL argument");
  if (h->host.bad_line != kNone) return pfail(C2V_ERR_STATE, "c2v_prep_assemble: the chunk has a line that cannot be sampled");
  cudaStream_t s = (cudaStream_t)stream;
  PCHECK(fn, cudaSetDevice(h->device));
  const long long nl = h->host.long_lines, L = h->host.lines;
  const long long n_picks = pick_off[nl];
  if (pick_off[0] != 0 || n_picks < 0 || (n_picks && !picks))
    return pfail(C2V_ERR_INVALID, "c2v_prep_assemble: pick_off must run from 0 over [long lines + 1] entries");
  PCHECK(fn, grow(h, h->picks, (size_t)(n_picks + 1) * 4));
  PCHECK(fn, grow(h, h->pick_off, (size_t)(nl + 1) * 8));
  PCHECK(fn, grow(h, h->out_len, (size_t)(L + 1) * 8));
  PCHECK(fn, grow(h, h->out_off, (size_t)(L + 1) * 8));
  if (n_picks) PCHECK(fn, cudaMemcpyAsync(h->picks.p, picks, n_picks * 4, cudaMemcpyHostToDevice, s));
  PCHECK(fn, cudaMemcpyAsync(h->pick_off.p, pick_off, (nl + 1) * 8, cudaMemcpyHostToDevice, s));
  const Lines a = lines_of(h);
  const Picks pk{P<int32_t>(h->long_rank), P<int32_t>(h->picks), P<long long>(h->pick_off)};
  long long* len = P<long long>(h->out_len);
  long long* off = P<long long>(h->out_off);
  out_len_kernel<<<kBlocks, kWarps * 32, 0, s>>>(a, pk, len);
  PCHECK(fn, cudaGetLastError());
  PCHECK(fn, with_temp(h, [&](void* tmp, size_t& bytes) {
    return cub::DeviceScan::ExclusiveSum(tmp, bytes, len, off, L + 1, s);
  }));
  long long total = 0;
  PCHECK(fn, cudaMemcpyAsync(&total, off + L, 8, cudaMemcpyDeviceToHost, s));
  PCHECK(fn, cudaStreamSynchronize(s));
  PCHECK(fn, grow(h, h->out, (size_t)total + 1));
  assemble_kernel<<<kBlocks, kWarps * 32, 0, s>>>(a, pk, off, P<char>(h->out));
  PCHECK(fn, cudaGetLastError());
  *text = P<char>(h->out);
  *nbytes = total;
  return C2V_OK;
}
