// Native tensoriser for `.c2v` text (reference path_context_reader.py:184-228 + filter :153-177):
// a chunk of complete lines -> int32 index rows + float32 mask rows written straight into
// caller-provided (pinned) host buffers, multi-threaded over lines, with the three vocabularies
// held in open-addressing hash tables.  Replaces tf.data's CsvDataset -> string_split ->
// StaticHashTable.lookup chain; string<->index work stays on the host, as in the reference.
//
// C ABI (bound with ctypes in path_context_reader.py):
//   c2v_vocab_create / c2v_vocab_destroy
//   c2v_vocab_export (the tables, for the device reader)
//   c2v_parse_chunk
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <thread>
#include <functional>
#include <vector>

namespace {

inline uint64_t hash_bytes(const char* p, size_t n) {        // FNV-1a 64
  uint64_t h = 1469598103934665603ull;
  for (size_t i = 0; i < n; ++i) { h ^= (unsigned char)p[i]; h *= 1099511628211ull; }
  return h ? h : 1;
}

struct Vocab {
  std::vector<char> bytes;            // all words, concatenated
  struct Slot { uint64_t h; int64_t off; int32_t len; int32_t idx; };
  std::vector<Slot> slots;            // h == 0: empty
  uint64_t mask = 0;
  int32_t oov = 0, pad = 0;

  int32_t lookup(const char* p, size_t n) const {
    const uint64_t h = hash_bytes(p, n);
    for (uint64_t i = h & mask;; i = (i + 1) & mask) {
      const Slot& s = slots[i];
      if (s.h == 0) return oov;
      if (s.h == h && (size_t)s.len == n && memcmp(bytes.data() + s.off, p, n) == 0) return s.idx;
    }
  }
};

struct ParseJob {
  const char* text;
  const int64_t* line_off;     // [n_lines + 1]
  int64_t n_lines;
  int C;
  const Vocab *tok, *pth, *tgt;
  int32_t *src, *path, *dst, *target;
  float* mask;
  uint8_t* keep;               // per line: 1 = passes the row filter
  int64_t* tgt_off;            // per line: offset / length of the target field (for evaluation strings)
  int32_t* tgt_len;
  int mode;                    // 0 train, 1 evaluate, 2 predict (no filter)
  std::atomic<int64_t> bad_line{-1};
  std::atomic<int> bad_kind{0};
};

// One pending vocabulary lookup of a line: the bytes of a context part, its hash, and -- once probed --
// the slot that may hold it.
struct Part {
  const char* p;
  uint32_t len;
  int32_t result;              // filled in by resolve()
  uint64_t h;
  const Vocab::Slot* cand;     // first slot with the same hash and length (nullptr: an empty slot came first)
};

// Lookups are latency-bound (two dependent cache misses each: the slot, then the word's bytes; the tables
// of a java14m-sized vocabulary are ~100 MB), so a line's ~600 lookups are issued as a software pipeline:
// hash every part and prefetch its slot, then probe all slots and prefetch the candidates' bytes, then compare.
inline void hash_and_prefetch(const Vocab& v, Part& q) {
  q.h = hash_bytes(q.p, q.len);
  __builtin_prefetch(&v.slots[q.h & v.mask]);
}

inline void probe(const Vocab& v, Part& q) {
  q.cand = nullptr;
  for (uint64_t i = q.h & v.mask;; i = (i + 1) & v.mask) {
    const Vocab::Slot& s = v.slots[i];
    if (s.h == 0) return;
    if (s.h == q.h && (uint32_t)s.len == q.len) {
      q.cand = &s;
      __builtin_prefetch(v.bytes.data() + s.off);
      return;
    }
  }
}

inline void resolve(const Vocab& v, Part& q) {
  if (!q.cand) { q.result = v.oov; return; }
  if (memcmp(v.bytes.data() + q.cand->off, q.p, q.len) == 0) { q.result = q.cand->idx; return; }
  q.result = v.lookup(q.p, q.len);        // same hash and length, different word: take the plain path
}

// one line -> one row.  Returns 0 ok, 1 wrong field count, 2 context with more than 3 parts.
// `parts` is per-thread scratch with room for 3 * C entries.
int parse_line(const ParseJob& J, int64_t li, Part* parts) {
  const char* p = J.text + J.line_off[li];
  const char* end = J.text + J.line_off[li + 1];
  while (end > p && (end[-1] == '\n' || end[-1] == '\r')) --end;
  const int C = J.C;
  int32_t* src = J.src + li * C;
  int32_t* pth = J.path + li * C;
  int32_t* dst = J.dst + li * C;
  float* msk = J.mask + li * C;
  const int32_t tpad = J.tok->pad, ppad = J.pth->pad;
  // field 0: target name
  const char* f = p;
  const char* sp = (const char*)memchr(f, ' ', end - f);
  const char* fe = sp ? sp : end;
  J.tgt_off[li] = f - J.text;
  J.tgt_len[li] = (int32_t)(fe - f);
  const int32_t ty = (fe == f) ? J.tgt->oov : J.tgt->lookup(f, fe - f);
  J.target[li] = ty;
  // pass 1: split the contexts; a part that is absent keeps len == UINT32_MAX and resolves to PAD
  constexpr uint32_t kAbsent = UINT32_MAX;
  int nfields = 1;
  int c = 0;
  while (sp) {
    f = sp + 1;
    sp = (const char*)memchr(f, ' ', end - f);
    fe = sp ? sp : end;
    ++nfields;
    if (c >= C) continue;       // keep counting fields for the error check
    Part* q = parts + 3 * c;
    q[0].len = q[1].len = q[2].len = kAbsent;
    if (fe != f) {
      const char* c1 = (const char*)memchr(f, ',', fe - f);
      if (!c1) {
        q[0].p = f; q[0].len = (uint32_t)(fe - f);                      // missing parts stay PAD
      } else {
        q[0].p = f; q[0].len = (uint32_t)(c1 - f);
        const char* c2 = (const char*)memchr(c1 + 1, ',', fe - (c1 + 1));
        if (!c2) {
          q[1].p = c1 + 1; q[1].len = (uint32_t)(fe - (c1 + 1));
        } else {
          q[1].p = c1 + 1; q[1].len = (uint32_t)(c2 - (c1 + 1));
          if (memchr(c2 + 1, ',', fe - (c2 + 1))) return 2;
          q[2].p = c2 + 1; q[2].len = (uint32_t)(fe - (c2 + 1));
        }
      }
      if (q[0].len != kAbsent) hash_and_prefetch(*J.tok, q[0]);
      if (q[1].len != kAbsent) hash_and_prefetch(*J.pth, q[1]);
      if (q[2].len != kAbsent) hash_and_prefetch(*J.tok, q[2]);
    }
    ++c;
  }
  if (nfields != C + 1) return 1;
  // pass 2: probe the (prefetched) slots, prefetch the candidates' bytes; pass 3: compare
  for (int i = 0; i < c; ++i) {
    Part* q = parts + 3 * i;
    if (q[0].len != kAbsent) probe(*J.tok, q[0]);
    if (q[1].len != kAbsent) probe(*J.pth, q[1]);
    if (q[2].len != kAbsent) probe(*J.tok, q[2]);
  }
  int32_t max_s = INT32_MIN, max_t = INT32_MIN, max_p = INT32_MIN;
  for (int i = 0; i < c; ++i) {
    Part* q = parts + 3 * i;
    int32_t s = tpad, k = ppad, t = tpad;
    if (q[0].len != kAbsent) { resolve(*J.tok, q[0]); s = q[0].result; }
    if (q[1].len != kAbsent) { resolve(*J.pth, q[1]); k = q[1].result; }
    if (q[2].len != kAbsent) { resolve(*J.tok, q[2]); t = q[2].result; }
    src[i] = s; pth[i] = k; dst[i] = t;
    msk[i] = (s != tpad || t != tpad || k != ppad) ? 1.0f : 0.0f;
    if (s > max_s) max_s = s;
    if (t > max_t) max_t = t;
    if (k > max_p) max_p = k;
  }
  // row filter (path_context_reader.py:153-177): reduce_max(indices) != PAD index, target > OOV (train)
  const bool any_valid = (max_s != tpad) || (max_t != tpad) || (max_p != ppad);
  uint8_t keep = 1;
  if (J.mode == 0) keep = (any_valid && ty > J.tgt->oov) ? 1 : 0;
  else if (J.mode == 1) keep = any_valid ? 1 : 0;
  J.keep[li] = keep;
  return 0;
}

}  // namespace

extern "C" {

// words: concatenated bytes; offsets: [n + 1]; indices: [n].  Duplicate words: the last one wins
// (as a Python dict built in order would).
void* c2v_vocab_create(const char* words, const int64_t* offsets, const int32_t* indices, int64_t n, int32_t oov, int32_t pad) {
  Vocab* v = new Vocab();
  v->oov = oov; v->pad = pad;
  v->bytes.assign(words, words + offsets[n]);
  uint64_t cap = 16;
  while (cap < (uint64_t)n * 2 + 2) cap <<= 1;
  v->slots.assign(cap, Vocab::Slot{0, 0, 0, 0});
  v->mask = cap - 1;
  for (int64_t i = 0; i < n; ++i) {
    const char* p = words + offsets[i];
    const size_t len = (size_t)(offsets[i + 1] - offsets[i]);
    const uint64_t h = hash_bytes(p, len);
    for (uint64_t j = h & v->mask;; j = (j + 1) & v->mask) {
      Vocab::Slot& s = v->slots[j];
      if (s.h == 0) { s = Vocab::Slot{h, offsets[i], (int32_t)len, indices[i]}; break; }
      if (s.h == h && (size_t)s.len == len && memcmp(v->bytes.data() + s.off, p, len) == 0) { s.idx = indices[i]; break; }
    }
  }
  return v;
}

void c2v_vocab_destroy(void* v) { delete (Vocab*)v; }

int32_t c2v_vocab_lookup(const void* v, const char* word, int64_t len) { return ((const Vocab*)v)->lookup(word, (size_t)len); }

// The table as it is, for the device reader (c2v_b200.h c2v_reader_vocab): *slots -> mask + 1 slots of 24 bytes
// {uint64 h, int64 off, int32 len, int32 idx} (h == 0: empty), *bytes -> the words' bytes (*n_bytes of them), and the
// OOV / PAD indices.  The pointers stay valid until c2v_vocab_destroy.
void c2v_vocab_export(const void* vp, const void** slots, uint64_t* mask, const char** bytes, int64_t* n_bytes,
                      int32_t* oov, int32_t* pad) {
  static_assert(sizeof(Vocab::Slot) == 24, "the device reader reads 24-byte slots");
  const Vocab* v = (const Vocab*)vp;
  *slots = v->slots.data();
  *mask = v->mask;
  *bytes = v->bytes.data();
  *n_bytes = (int64_t)v->bytes.size();
  *oov = v->oov;
  *pad = v->pad;
}

// Parses the complete lines in text[0, len) (the last line may lack a trailing newline).
// Outputs hold one row per line, in line order: src/path/dst [n, C] int32, mask [n, C] float32,
// target [n] int32, keep [n] uint8 (row filter), tgt_off/tgt_len [n] (target field location).
// Returns the number of lines (<= capacity), or -(line number + 1) on a malformed line with
// *err_kind = 1 (field count) / 2 (context with > 3 parts), or INT64_MIN if capacity is too small.
// Blank lines are skipped (they still count in the reported line number).
int64_t c2v_parse_chunk(const char* text, int64_t len, int32_t max_contexts, const void* tok, const void* pth, const void* tgt,
                        int32_t mode, int32_t n_threads, int64_t capacity, int32_t* src, int32_t* path, int32_t* dst,
                        float* mask, int32_t* target, uint8_t* keep, int64_t* tgt_off, int32_t* tgt_len, int32_t* err_kind) {
  // blank lines ("" / "\n") are not records: the Python statement of the reader skips them too.  A record's span
  // runs to the next record's start, so blank lines after it are trimmed with its own newline.
  std::vector<int64_t> off, lineno;
  off.reserve(1024);
  lineno.reserve(1024);
  int64_t pos = 0, line = 0;
  while (pos < len) {
    const char* nl = (const char*)memchr(text + pos, '\n', len - pos);
    const int64_t next = nl ? (nl - text) + 1 : len;
    if (!(nl && nl == text + pos)) { off.push_back(pos); lineno.push_back(line); }
    pos = next;
    ++line;
  }
  off.push_back(len);
  const int64_t n = (int64_t)off.size() - 1;
  if (n > capacity) return INT64_MIN;
  ParseJob J;
  J.text = text; J.line_off = off.data(); J.n_lines = n; J.C = max_contexts;
  J.tok = (const Vocab*)tok; J.pth = (const Vocab*)pth; J.tgt = (const Vocab*)tgt;
  J.src = src; J.path = path; J.dst = dst; J.mask = mask; J.target = target; J.keep = keep;
  J.tgt_off = tgt_off; J.tgt_len = tgt_len; J.mode = mode;
  if (n_threads < 1) n_threads = 1;
  if (n_threads > 64) n_threads = 64;
  if ((int64_t)n_threads > n) n_threads = n > 0 ? (int)n : 1;
  auto work = [&](int t) {
    const int64_t lo = n * t / n_threads, hi = n * (t + 1) / n_threads;
    std::vector<Part> parts((size_t)3 * (max_contexts > 0 ? max_contexts : 1));
    for (int64_t i = lo; i < hi; ++i) {
      const int rc = parse_line(J, i, parts.data());
      if (rc) {
        int64_t expect = -1;
        if (J.bad_line.compare_exchange_strong(expect, i)) J.bad_kind.store(rc);
        return;
      }
    }
  };
  if (n_threads == 1) {
    work(0);
  } else {
    std::vector<std::thread> th;
    for (int t = 0; t < n_threads; ++t) th.emplace_back(work, t);
    for (auto& x : th) x.join();
  }
  if (J.bad_line.load() >= 0) {
    if (err_kind) *err_kind = J.bad_kind.load();
    return -(lineno[(size_t)J.bad_line.load()] + 1);
  }
  return n;
}

// Shuffle-pool draw (path_context_reader._RowPool.take) over the five parallel row arrays of the pool -- src / path / dst [cap, C]
// int32, mask [cap, C] float32, target [cap] int32, of which rows [0, n) are live.  Rows pick[0..b) are copied to the out buffers in
// pick order; the holes they leave below the new end n - b are then filled with the surviving rows of the tail [n - b, n), both in
// ascending order -- the numpy statement is  holes = flatnonzero(chosen[:n-b]); movers = n-b + flatnonzero(~chosen[n-b:]);
// a[holes] = a[movers].  Row copies are spread over n_threads.  Returns 0, or -1 if pick is not b distinct indices in [0, n).
int32_t c2v_pool_take(int32_t* src, int32_t* path, int32_t* dst, float* mask, int32_t* target, int64_t n, int32_t C,
                      const int64_t* pick, int32_t b, int32_t* o_src, int32_t* o_path, int32_t* o_dst, float* o_mask,
                      int32_t* o_target, int32_t n_threads) {
  if (b < 0 || b > n || C < 1) return -1;
  std::vector<uint8_t> chosen((size_t)n, 0);
  for (int32_t i = 0; i < b; ++i) {
    const int64_t r = pick[i];
    if (r < 0 || r >= n || chosen[(size_t)r]) return -1;
    chosen[(size_t)r] = 1;
  }
  const int64_t new_n = n - b;
  std::vector<int64_t> holes, movers;
  holes.reserve((size_t)b);
  movers.reserve((size_t)b);
  for (int64_t r = 0; r < new_n; ++r)
    if (chosen[(size_t)r]) holes.push_back(r);
  for (int64_t r = new_n; r < n; ++r)
    if (!chosen[(size_t)r]) movers.push_back(r);
  const size_t row = (size_t)C * 4;
  if (n_threads < 1) n_threads = 1;
  if (n_threads > 16) n_threads = 16;
  auto spread = [&](int64_t count, const std::function<void(int64_t, int64_t)>& body) {
    const int t_n = (int)std::min<int64_t>(n_threads, std::max<int64_t>(count / 64, 1));
    if (t_n <= 1) { body(0, count); return; }
    std::vector<std::thread> th;
    for (int t = 0; t < t_n; ++t) th.emplace_back(body, count * t / t_n, count * (t + 1) / t_n);
    for (auto& x : th) x.join();
  };
  // the copies are random 4 x (C * 4)-byte rows out of tens of MB: latency-bound, so the rows a few iterations ahead are
  // prefetched (every cache line of them) while the current one is copied
  auto prefetch_row = [&](size_t r) {
    for (size_t o = 0; o < row; o += 64) {
      __builtin_prefetch((const char*)(src + r * C) + o);
      __builtin_prefetch((const char*)(path + r * C) + o);
      __builtin_prefetch((const char*)(dst + r * C) + o);
      __builtin_prefetch((const char*)(mask + r * C) + o);
    }
  };
  constexpr int64_t kAhead = 4;
  spread(b, [&](int64_t lo, int64_t hi) {
    for (int64_t i = lo; i < std::min(lo + kAhead, hi); ++i) prefetch_row((size_t)pick[i]);
    for (int64_t i = lo; i < hi; ++i) {
      if (i + kAhead < hi) prefetch_row((size_t)pick[i + kAhead]);
      const size_t r = (size_t)pick[i];
      memcpy(o_src + (size_t)i * C, src + r * C, row);
      memcpy(o_path + (size_t)i * C, path + r * C, row);
      memcpy(o_dst + (size_t)i * C, dst + r * C, row);
      memcpy(o_mask + (size_t)i * C, mask + r * C, row);
      o_target[i] = target[r];
    }
  });
  // every picked row has been copied out before any hole is overwritten (spread() joins its threads)
  spread((int64_t)holes.size(), [&](int64_t lo, int64_t hi) {
    for (int64_t i = lo; i < std::min(lo + kAhead, hi); ++i) prefetch_row((size_t)movers[(size_t)i]);
    for (int64_t i = lo; i < hi; ++i) {
      if (i + kAhead < hi) prefetch_row((size_t)movers[(size_t)(i + kAhead)]);
      const size_t h = (size_t)holes[(size_t)i], m = (size_t)movers[(size_t)i];
      memcpy(src + h * C, src + m * C, row);
      memcpy(path + h * C, path + m * C, row);
      memcpy(dst + h * C, dst + m * C, row);
      memcpy(mask + h * C, mask + m * C, row);
      target[h] = target[m];
    }
  });
  return 0;
}

}  // extern "C"
