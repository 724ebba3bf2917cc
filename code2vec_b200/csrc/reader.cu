// Device reader of `.c2v` training text (include/c2v_b200.h "Device reader", DESIGN.md §6d): a chunk of complete lines
// already in device memory -> rows of the training shuffle pool, and draws from that pool into device batch buffers.
// It computes what the host tensoriser computes (native/batcher.cpp parse_line, c2v_pool_take) and what the host
// reader's shuffle pool does with it (path_context_reader._RowPool.commit / take), so its batches are the host reader's
// batches, bit for bit:
//   line index : per-tile counts of record starts and newlines, one-block scans, then each record's byte offset and the
//                number of its line (blank lines are skipped but keep their line numbers, as the host's errors count them)
//   parse      : one warp per record; fields are split on ' ' and parts on ',' with ballots, each part is hashed
//                (FNV-1a 64) by one lane and probed in the host's own open-addressing tables, bytes compared
//   commit     : rows land behind the pool's live end; dropped rows below the kept count are filled by the kept rows
//                beyond it, j-th hole from j-th mover (not a stable compaction: the host pool's order)
//   draw       : the picked rows (the host's random draw) are gathered into a batch buffer, then the holes they leave
//                below the new end are filled with the surviving tail rows, both in ascending order
// A chunk read sharded across ranks (DESIGN.md §6d) runs the line index and the parse over one rank's share of the chunk
// into a peer-visible stage; every rank then copies all stages behind its pool's live end in rank order (assemble) and
// commits the whole chunk's records as above, so its pool is the one a whole-chunk parse builds.
// Test files (DESIGN.md §6e) take the same line index and parse with the evaluate filter; their kept records go to an
// evaluation queue in file order with their names, and eval_score_kernel scores the engine's top-k ids of a batch.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <string>

#include "../../include/c2v_b200.h"
#include "vocab_lookup.cuh"

namespace c2v {
void set_global_error(const std::string& msg);     // engine.cu: the message c2v_last_error(NULL) returns
}

namespace {

constexpr int kTile = 4096;                        // bytes per block of the line index
constexpr int kTileThreads = 256;
constexpr int kPerThread = kTile / kTileThreads;
constexpr int kRowTile = 1024;                     // rows per block of the commit scan
constexpr int kParseWarps = 4;
constexpr unsigned kFull = 0xffffffffu;

// ---- line index ----------------------------------------------------------------------------------------------------
// a record starts at byte p when p == 0 or text[p-1] == '\n', unless text[p] is '\n' itself (a blank line)
__device__ __forceinline__ void count_bytes(const unsigned char* text, long long n, long long lo, int& recs, int& nls) {
  recs = nls = 0;
  for (int k = 0; k < kPerThread; ++k) {
    const long long p = lo + k;
    if (p >= n) break;
    const unsigned char c = text[p];
    recs += (p == 0 || text[p - 1] == '\n') && c != '\n';
    nls += c == '\n';
  }
}

__global__ void __launch_bounds__(kTileThreads)
line_count_kernel(const unsigned char* __restrict__ text, long long n, int* __restrict__ rec_cnt, int* __restrict__ nl_cnt) {
  using Reduce = cub::BlockReduce<long long, kTileThreads>;
  __shared__ typename Reduce::TempStorage tmp;
  int r, l;
  count_bytes(text, n, (long long)blockIdx.x * kTile + threadIdx.x * kPerThread, r, l);
  const long long s = Reduce(tmp).Sum(((long long)r << 32) | l);      // both counts are <= kTile: no carry between halves
  if (threadIdx.x == 0) {
    rec_cnt[blockIdx.x] = (int)(s >> 32);
    nl_cnt[blockIdx.x] = (int)(s & 0xffffffff);
  }
}

// exclusive scan of in[0, n) into out[0, n), out[n] = the total (one block)
__global__ void __launch_bounds__(1024) exclusive_scan_kernel(const int* __restrict__ in, int* __restrict__ out, int n) {
  using Scan = cub::BlockScan<int, 1024>;
  __shared__ typename Scan::TempStorage tmp;
  const int per = (n + 1023) / 1024;
  const int lo = min(n, (int)threadIdx.x * per), hi = min(n, lo + per);
  int s = 0;
  for (int i = lo; i < hi; ++i) s += in[i];
  int run, total;
  Scan(tmp).ExclusiveSum(s, run, total);
  for (int i = lo; i < hi; ++i) {
    out[i] = run;
    run += in[i];
  }
  if (threadIdx.x == 0) out[n] = total;
}

// rec_off[i] = first byte of record i, rec_line[i] = its line number (newlines before it), for the first `cap` records
__global__ void __launch_bounds__(kTileThreads)
line_index_kernel(const unsigned char* __restrict__ text, long long n, const int* __restrict__ rec_base,
                  const int* __restrict__ nl_base, long long cap, long long* __restrict__ rec_off,
                  long long* __restrict__ rec_line) {
  using Scan = cub::BlockScan<long long, kTileThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const long long lo = (long long)blockIdx.x * kTile + threadIdx.x * kPerThread;
  int r, l;
  count_bytes(text, n, lo, r, l);
  long long before;
  Scan(tmp).ExclusiveSum(((long long)r << 32) | l, before);
  long long rec = rec_base[blockIdx.x] + (before >> 32);
  long long line = nl_base[blockIdx.x] + (before & 0xffffffff);
  for (int k = 0; k < kPerThread; ++k) {
    const long long p = lo + k;
    if (p >= n) break;
    const unsigned char c = text[p];
    if ((p == 0 || text[p - 1] == '\n') && c != '\n') {
      if (rec < cap) { rec_off[rec] = p; rec_line[rec] = line; }
      ++rec;
    }
    line += c == '\n';
  }
}

// ---- parse ---------------------------------------------------------------------------------------------------------
struct ParseArgs {
  const unsigned char* text;
  long long nbytes;
  int C;
  DevVocab tok, pth, tgt;
  const long long* rec_off;
  const int* n_rec;               // records in the chunk (line_count scan total)
  long long cap;                  // rows reserved behind the pool's end
  int32_t *src, *path, *dst, *target;     // pool rows from the live end
  float* mask;
  uint8_t* keep;                  // per record: passes the filter of `mode`
  unsigned long long* bad;        // lowest malformed record << 2 | kind
  int mode;                       // 0: training filter (a valid context and target > OOV), 1: evaluate (a valid context)
  int* name_len;                  // evaluate: per record, the bytes of field 0 (the name; 0 = empty); NULL in training
};

// a part that ends at a separator: part kk of context field f, bytes [start, start + len) of the line
__device__ __forceinline__ void note_part(longlong2* parts, int C, long long f, int kk, long long start, long long len,
                                          bool by_space) {
  if (f < 1 || f > C || kk > 2) return;
  if (by_space && kk == 0 && len == 0) return;        // an empty context: all three parts stay absent (PAD)
  parts[(f - 1) * 3 + kk] = make_longlong2(start, len);
}

__global__ void __launch_bounds__(32 * kParseWarps) parse_kernel(const __grid_constant__ ParseArgs a) {
  extern __shared__ longlong2 shm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int C = a.C;
  longlong2* parts = shm + (size_t)warp * 3 * C;       // per part: (start, len), len -1 = absent
  const long long R = min((long long)*a.n_rec, a.cap);
  const unsigned lt = (1u << lane) - 1;
  for (long long li = (long long)blockIdx.x * kParseWarps + warp; li < R; li += (long long)gridDim.x * kParseWarps) {
    const long long b0 = a.rec_off[li];
    long long e = li + 1 < R ? a.rec_off[li + 1] : a.nbytes;     // a record runs to the next one (blank lines included)
    const unsigned char* p = a.text + b0;
    while (e > b0 && (a.text[e - 1] == '\n' || a.text[e - 1] == '\r')) --e;
    const long long len = e - b0;
    for (int i = lane; i < 3 * C; i += 32) parts[i] = make_longlong2(0, -1);
    __syncwarp();
    long long f = 0;              // spaces before the window: the field the window starts in
    int k = 0;                    // context commas since the current field began
    long long last = -1;          // the last separator before the window
    long long tgt_len = -1;       // length of field 0 (the target) once its space is seen
    bool bad3 = false;            // a context among the first C has a third comma
    for (long long w = 0; w < len; w += 32) {
      const long long pos = w + lane;
      const unsigned char c = pos < len ? p[pos] : 0;
      const unsigned sp = __ballot_sync(kFull, c == ' ');
      const long long f_here = f + __popc(sp & lt);
      const unsigned cm = __ballot_sync(kFull, c == ',' && f_here >= 1);     // commas inside field 0 are target bytes
      const unsigned sep = sp | cm;
      if ((sep >> lane) & 1) {
        const unsigned before = sep & lt;
        const long long start = before ? w + (31 - __clz(before)) + 1 : last + 1;
        const unsigned sp_before = sp & lt;
        int kk;
        if (sp_before) {
          const int ls = 31 - __clz(sp_before);
          kk = __popc(cm & lt & ~((2u << ls) - 1u));
        } else {
          kk = k + __popc(cm & lt);
        }
        if (c == ',' && kk >= 2 && f_here <= C) bad3 = true;
        note_part(parts, C, f_here, kk, start, pos - start, c == ' ');
      }
      if (f == 0 && sp) tgt_len = w + __ffs(sp) - 1;
      if (sep) last = w + (31 - __clz(sep));
      if (sp) {
        const int ls = 31 - __clz(sp);
        k = __popc(cm & ~((2u << ls) - 1u));
      } else {
        k += __popc(cm);
      }
      f += __popc(sp);
    }
    if (lane == 0 && f >= 1) note_part(parts, C, f, k, last + 1, len - last - 1, true);    // the line's last part
    const bool any3 = __any_sync(kFull, bad3);
    const int kind = any3 ? 2 : (f + 1 != C + 1 ? 1 : 0);
    if (kind) {
      if (lane == 0) atomicMin(a.bad, ((unsigned long long)li << 2) | (unsigned long long)kind);
      __syncwarp();
      continue;
    }
    if (tgt_len < 0) tgt_len = len;
    __syncwarp();
    for (int i = lane; i < 3 * C; i += 32) {
      const longlong2 q = parts[i];
      const DevVocab& v = (i % 3 == 1) ? a.pth : a.tok;
      const int32_t r = q.y < 0 ? v.pad : lookup(v, p + q.x, q.y);
      parts[i].x = r;
    }
    int32_t ty = 0;
    if (lane == 0) ty = tgt_len == 0 ? a.tgt.oov : lookup(a.tgt, p, tgt_len);
    __syncwarp();
    const long long row = li * C;
    int max_s = INT32_MIN, max_p = INT32_MIN, max_t = INT32_MIN;
    for (int c = lane; c < C; c += 32) {
      const int32_t s = (int32_t)parts[3 * c].x, q = (int32_t)parts[3 * c + 1].x, t = (int32_t)parts[3 * c + 2].x;
      a.src[row + c] = s;
      a.path[row + c] = q;
      a.dst[row + c] = t;
      a.mask[row + c] = (s != a.tok.pad || t != a.tok.pad || q != a.pth.pad) ? 1.0f : 0.0f;
      max_s = max(max_s, s);
      max_p = max(max_p, q);
      max_t = max(max_t, t);
    }
    max_s = __reduce_max_sync(kFull, max_s);
    max_p = __reduce_max_sync(kFull, max_p);
    max_t = __reduce_max_sync(kFull, max_t);
    if (lane == 0) {
      const bool any_valid = max_s != a.tok.pad || max_t != a.tok.pad || max_p != a.pth.pad;
      a.target[li] = ty;
      a.keep[li] = (any_valid && (a.mode == 1 || ty > a.tgt.oov)) ? 1 : 0;
      if (a.name_len) a.name_len[li] = (int)tgt_len;
    }
    __syncwarp();
  }
}

// ---- pool commit -----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) keep_count_kernel(const uint8_t* __restrict__ keep, const int* __restrict__ n_rec,
                                                         long long cap, int* __restrict__ cnt) {
  using Reduce = cub::BlockReduce<int, 256>;
  __shared__ typename Reduce::TempStorage tmp;
  const long long R = min((long long)*n_rec, cap);
  const long long lo = (long long)blockIdx.x * kRowTile + threadIdx.x * 4;
  int s = 0;
  for (int k = 0; k < 4; ++k) s += (lo + k < R) ? keep[lo + k] : 0;
  s = Reduce(tmp).Sum(s);
  if (threadIdx.x == 0) cnt[blockIdx.x] = s;
}

// holes[j] = the j-th dropped row below the kept count, movers[j] = the j-th kept row at or beyond it (_RowPool.commit);
// *n_moves = their number.  K(i) = kept rows before row i; kept = K(R).
__global__ void __launch_bounds__(256)
commit_index_kernel(const uint8_t* __restrict__ keep, const int* __restrict__ n_rec, long long cap,
                    const int* __restrict__ base, int tiles, int* __restrict__ holes, int* __restrict__ movers,
                    int* __restrict__ n_moves) {
  using Scan = cub::BlockScan<int, 256>;
  using Reduce = cub::BlockReduce<int, 256>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ typename Reduce::TempStorage rtmp;
  __shared__ int Kk_shared;
  const long long R = min((long long)*n_rec, cap);
  const int kept = base[tiles];
  // K(kept): the kept rows below the kept count
  const int tk = kept / kRowTile;
  int part = 0;
  for (long long i = (long long)tk * kRowTile + threadIdx.x; i < kept; i += 256) part += keep[i];
  part = Reduce(rtmp).Sum(part);                 // valid in thread 0 only
  if (threadIdx.x == 0) Kk_shared = (tk < tiles ? base[tk] : kept) + part;
  __syncthreads();
  const int Kk = Kk_shared;
  const long long lo = (long long)blockIdx.x * kRowTile + threadIdx.x * 4;
  int s = 0;
  for (int k = 0; k < 4; ++k) s += (lo + k < R) ? keep[lo + k] : 0;
  int K;
  Scan(tmp).ExclusiveSum(s, K);
  K += base[blockIdx.x];
  for (int k = 0; k < 4; ++k) {
    const long long i = lo + k;
    if (i >= R) break;
    const int kp = keep[i];
    if (i < kept && !kp) holes[i - K] = (int)i;
    if (i >= kept && kp) movers[K - Kk] = (int)i;
    K += kp;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *n_moves = kept - Kk;
}

struct PoolRows {
  int32_t *src, *path, *dst, *target;
  float* mask;
};

// pool row to[j] <- pool row from[j] for j < *count (one warp per row; the two index sets are disjoint)
__global__ void __launch_bounds__(256)
move_rows_kernel(PoolRows pool, int C, long long row0, const int* __restrict__ to, const int* __restrict__ from,
                 const int* __restrict__ count) {
  const int n = *count;
  const int lane = threadIdx.x & 31;
  for (long long j = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5; j < n; j += ((long long)gridDim.x * 256) >> 5) {
    const long long d = (row0 + to[j]) * C, s = (row0 + from[j]) * C;
    for (int c = lane; c < C; c += 32) {
      pool.src[d + c] = pool.src[s + c];
      pool.path[d + c] = pool.path[s + c];
      pool.dst[d + c] = pool.dst[s + c];
      pool.mask[d + c] = pool.mask[s + c];
    }
    if (lane == 0) pool.target[row0 + to[j]] = pool.target[row0 + from[j]];
  }
}

// ---- draw ------------------------------------------------------------------------------------------------------------
// c2v_pool_take's index sets, one block: holes = the picks below new_n in ascending order, movers = the rows of the tail
// [new_n, n) that were not picked, ascending.  tail: b bytes of scratch.
__global__ void __launch_bounds__(1024)
draw_index_kernel(const long long* __restrict__ pick, int b, long long n, uint8_t* __restrict__ tail,
                  int* __restrict__ holes, int* __restrict__ movers, int* __restrict__ n_moves) {
  using Scan = cub::BlockScan<int, 1024>;
  __shared__ typename Scan::TempStorage tmp;
  const long long new_n = n - b;
  for (int i = threadIdx.x; i < b; i += 1024) tail[i] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < b; i += 1024)
    if (pick[i] >= new_n) tail[pick[i] - new_n] = 1;
  __syncthreads();
  for (int i = threadIdx.x; i < b; i += 1024) {      // a pick's rank among the picks below new_n: how many are smaller
    const long long v = pick[i];
    if (v >= new_n) continue;
    int rank = 0;
    for (int q = 0; q < b; ++q) rank += pick[q] < v;
    holes[rank] = (int)v;
  }
  const int per = (b + 1023) / 1024;
  const int lo = min(b, (int)threadIdx.x * per), hi = min(b, lo + per);
  int s = 0;
  for (int i = lo; i < hi; ++i) s += !tail[i];
  int run, total;
  Scan(tmp).ExclusiveSum(s, run, total);
  for (int i = lo; i < hi; ++i)
    if (!tail[i]) movers[run++] = (int)(new_n + i);
  if (threadIdx.x == 0) *n_moves = total;
}

// out row i - lo <- pool row pick[i] for i in [lo, hi) (one warp per row)
__global__ void __launch_bounds__(256)
gather_kernel(PoolRows pool, int C, const long long* __restrict__ pick, int lo, int hi, PoolRows out) {
  const int lane = threadIdx.x & 31;
  for (long long i = lo + (((long long)blockIdx.x * 256 + threadIdx.x) >> 5); i < hi; i += ((long long)gridDim.x * 256) >> 5) {
    const long long r = pick[i], d = (i - lo) * C, s = r * C;
    for (int c = lane; c < C; c += 32) {
      out.src[d + c] = pool.src[s + c];
      out.path[d + c] = pool.path[s + c];
      out.dst[d + c] = pool.dst[s + c];
      out.mask[d + c] = pool.mask[s + c];
    }
    if (lane == 0) out.target[i - lo] = pool.target[r];
  }
}

// ---- sharded chunks --------------------------------------------------------------------------------------------------
// A stage of `rows` rows: the share's status (c2v_reader_share_status, its `rows` field included) in the first 256 bytes,
// then src, path, dst, mask [rows, C], target [rows] and keep [rows], each at a 256-byte boundary.
constexpr long long kStageHeader = 256;
constexpr int kMaxShares = 64;

struct StageLayout { long long src, path, dst, mask, target, keep, bytes; };

__host__ __device__ __forceinline__ long long align256(long long x) { return (x + 255) & ~255ll; }

__host__ __device__ __forceinline__ StageLayout stage_layout(int C, long long rows) {
  const long long m = align256(rows * C * 4);
  StageLayout L;
  L.src = kStageHeader;
  L.path = L.src + m;
  L.dst = L.path + m;
  L.mask = L.dst + m;
  L.target = L.mask + m;
  L.keep = L.target + align256(rows * 4);
  L.bytes = L.keep + align256(rows);
  return L;
}

struct ShareSrc {
  const unsigned char* stage;     // this rank's stage or a peer's, opened through CUDA IPC
  long long row0, records;        // first row of the share in the chunk, its records
};

struct AssembleArgs {
  ShareSrc share[kMaxShares];
  int n, C;
  PoolRows pool;
  long long live;                 // the pool's live end: the chunk's row 0
  uint8_t* keep;                  // per record of the chunk
  int* n_rec;                     // <- the chunk's records
  long long total;
};

// pool rows [live + row0, live + row0 + records) and keep[row0, row0 + records) <- stage blockIdx.y's rows and keep flags
__global__ void __launch_bounds__(256) assemble_shares_kernel(const __grid_constant__ AssembleArgs a) {
  __shared__ long long rows;
  const ShareSrc sh = a.share[blockIdx.y];
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *a.n_rec = (int)a.total;
  if (sh.records == 0) return;
  if (threadIdx.x == 0) rows = ((const c2v_reader_share_status*)sh.stage)->rows;
  __syncthreads();
  const StageLayout L = stage_layout(a.C, rows);
  const int32_t* src = (const int32_t*)(sh.stage + L.src);
  const int32_t* path = (const int32_t*)(sh.stage + L.path);
  const int32_t* dst = (const int32_t*)(sh.stage + L.dst);
  const float* mask = (const float*)(sh.stage + L.mask);
  const int32_t* target = (const int32_t*)(sh.stage + L.target);
  const uint8_t* keep = sh.stage + L.keep;
  const long long n = sh.records * a.C, d0 = (a.live + sh.row0) * a.C;
  const long long stride = (long long)gridDim.x * 256;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += stride) {
    const int32_t s = src[i], q = path[i], t = dst[i];
    const float m = mask[i];
    a.pool.src[d0 + i] = s;
    a.pool.path[d0 + i] = q;
    a.pool.dst[d0 + i] = t;
    a.pool.mask[d0 + i] = m;
  }
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < sh.records; i += stride) {
    a.pool.target[a.live + sh.row0 + i] = target[i];
    a.keep[sh.row0 + i] = keep[i];
  }
}

// ---- evaluation queue (c2v_reader_eval_*) --------------------------------------------------------------------------
// The kept records of a chunk parsed in evaluate mode, appended to a queue in file order (a stable compaction, unlike the
// pool commit), each with its name: field 0's bytes, or the target vocabulary's OOV word when field 0 is empty.

// movers[K] = i for the K-th kept record i (ascending); qlen[K] = its name's length, qlen[kept, cap) = 0
__global__ void __launch_bounds__(256)
eval_index_kernel(const uint8_t* __restrict__ keep, const int* __restrict__ n_rec, long long cap,
                  const int* __restrict__ base, int tiles, const int* __restrict__ name_len, int oov_len,
                  int* __restrict__ movers, int* __restrict__ qlen) {
  using Scan = cub::BlockScan<int, 256>;
  __shared__ typename Scan::TempStorage tmp;
  const long long R = min((long long)*n_rec, cap);
  const int kept = base[tiles];
  const long long lo = (long long)blockIdx.x * kRowTile + threadIdx.x * 4;
  int s = 0;
  for (int k = 0; k < 4; ++k) s += (lo + k < R) ? keep[lo + k] : 0;
  int K;
  Scan(tmp).ExclusiveSum(s, K);
  K += base[blockIdx.x];
  for (int k = 0; k < 4; ++k) {
    const long long i = lo + k;
    if (i < R && keep[i]) {
      movers[K] = (int)i;
      qlen[K] = name_len[i] > 0 ? name_len[i] : oov_len;
      ++K;
    }
    if (i >= kept && i < cap) qlen[i] = 0;
  }
}

struct EvalAppendArgs {
  PoolRows from, to;              // parsed records (pool room), queue rows from its end
  int C, kept;
  const int* movers;              // [kept] record of each appended row
  const int* qoff;                // [kept] name offset from names_end (scan of qlen)
  const long long* rec_off;       // record -> first byte in text
  const int* name_len;            // record -> bytes of field 0 (0: the OOV word)
  const unsigned char* text;
  const unsigned char* oov_word;  // the target OOV word (word table entry)
  int oov_len;
  long long names_end;            // arena bytes in use before the append
  unsigned char* names;
  long long* noff;                // name offsets from the queue's end row
  long long name_total;
};

// queue row j <- record movers[j], its name -> names[names_end + qoff[j]] (one warp per row)
__global__ void __launch_bounds__(256) eval_append_kernel(const __grid_constant__ EvalAppendArgs a) {
  const int lane = threadIdx.x & 31;
  for (long long j = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5; j < a.kept; j += ((long long)gridDim.x * 256) >> 5) {
    const int i = a.movers[j];
    const long long s = (long long)i * a.C, d = j * a.C;
    for (int c = lane; c < a.C; c += 32) {
      a.to.src[d + c] = a.from.src[s + c];
      a.to.path[d + c] = a.from.path[s + c];
      a.to.dst[d + c] = a.from.dst[s + c];
      a.to.mask[d + c] = a.from.mask[s + c];
    }
    const long long o = a.names_end + a.qoff[j];
    const long long n = (j + 1 < a.kept ? a.names_end + a.qoff[j + 1] : a.names_end + a.name_total) - o;
    const unsigned char* src = a.name_len[i] > 0 ? a.text + a.rec_off[i] : a.oov_word;
    for (long long b = lane; b < n; b += 32) a.names[o + b] = src[b];
    if (lane == 0) {
      a.to.target[j] = a.from.target[i];
      a.noff[j] = o;
      if (j + 1 == a.kept) a.noff[j + 1] = o + n;
    }
  }
}

// queue rows [head, head + n) -> [0, n), their names to the arena's front, offsets rebased (the two ranges are disjoint)
__global__ void __launch_bounds__(256)
eval_compact_kernel(PoolRows q, int C, long long head, long long n, long long* __restrict__ noff,
                    unsigned char* __restrict__ names) {
  const int lane = threadIdx.x & 31;
  const long long nh = noff[head];
  for (long long j = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5; j < n; j += ((long long)gridDim.x * 256) >> 5) {
    const long long s = (head + j) * C, d = j * C;
    for (int c = lane; c < C; c += 32) {
      q.src[d + c] = q.src[s + c];
      q.path[d + c] = q.path[s + c];
      q.dst[d + c] = q.dst[s + c];
      q.mask[d + c] = q.mask[s + c];
    }
    const long long o = noff[head + j], e = noff[head + j + 1];
    for (long long b = lane; b < e - o; b += 32) names[o - nh + b] = names[o + b];
    if (lane == 0) {
      q.target[j] = q.target[head + j];
      noff[j] = o - nh;
      if (j + 1 == n) noff[j + 1] = e - nh;
    }
  }
}

// out row j <- queue row head + j, its name -> out_names[out_off[j]] (offsets from the batch's first name; one warp a row)
__global__ void __launch_bounds__(256)
eval_take_kernel(PoolRows q, int C, long long head, int b, const long long* __restrict__ noff,
                 const unsigned char* __restrict__ names, PoolRows out, long long* __restrict__ out_off,
                 unsigned char* __restrict__ out_names, long long names_cap) {
  const int lane = threadIdx.x & 31;
  const long long nh = noff[head];
  for (long long j = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5; j < b; j += ((long long)gridDim.x * 256) >> 5) {
    const long long s = (head + j) * C, d = j * C;
    for (int c = lane; c < C; c += 32) {
      out.src[d + c] = q.src[s + c];
      out.path[d + c] = q.path[s + c];
      out.dst[d + c] = q.dst[s + c];
      out.mask[d + c] = q.mask[s + c];
    }
    const long long o = noff[head + j], e = noff[head + j + 1];
    for (long long x = lane; x < e - o && o - nh + x < names_cap; x += 32) out_names[o - nh + x] = names[o + x];
    if (lane == 0) {
      out.target[j] = q.target[head + j];
      out_off[j] = o - nh;
      if (j + 1 == b) out_off[j + 1] = e - nh;
    }
  }
}

// ---- evaluation metrics (c2v_reader_eval_score) ----------------------------------------------------------------------
struct EvalTables {
  const unsigned char* words;     // target words, concatenated; word_off [Y + 1]
  const long long* word_off;
  const unsigned char* norm;      // normalize_word of each word; norm_off [Y + 1]
  const long long* norm_off;
  const uint8_t* legal;           // legal_method_names_checker of each word
  int Y;
};

__device__ __forceinline__ bool ascii_letter(unsigned char c) { return (unsigned char)((c | 0x20) - 'a') < 26; }

// normalize_word(name) == nw[0, m) for an ASCII name: its letters lowercased, or the name itself when it has none
__device__ bool norm_equal(const unsigned char* name, long long L, bool letters, const unsigned char* nw, long long m) {
  if (!letters) {
    if (L != m) return false;
    for (long long p = 0; p < L; ++p)
      if (name[p] != nw[p]) return false;
    return true;
  }
  long long j = 0;
  for (long long p = 0; p < L; ++p) {
    const unsigned char c = name[p];
    if (!ascii_letter(c)) continue;
    if (j >= m || (unsigned char)(c | 0x20) != nw[j]) return false;
    ++j;
  }
  return j == m;
}

// the j-th '|'-separated subtoken of s[0, L) (empty ones count): *start, returns its length
__device__ long long subtoken(const unsigned char* s, long long L, long long j, long long* start) {
  long long p = 0;
  for (long long t = 0; t < j; ++p)
    if (s[p] == '|') ++t;
  long long e = p;
  while (e < L && s[e] != '|') ++e;
  *start = p;
  return e - p;
}

// whether t[0, tl) is one of the subtokens of s[0, L)
__device__ bool has_subtoken(const unsigned char* s, long long L, const unsigned char* t, long long tl) {
  long long start = 0;
  for (long long p = 0; p <= L; ++p) {
    if (p < L && s[p] != '|') continue;
    if (p - start == tl) {
      long long q = 0;
      while (q < tl && s[start + q] == t[q]) ++q;
      if (q == tl) return true;
    }
    start = p + 1;
  }
  return false;
}

// One warp per row: the rank of the first match among the legal words of the row's top-k (get_first_match_word_from_
// top_predictions), the first legal word, and the subtoken counts of that word against the name
// (SubtokensEvaluationMetric.update_batch).  Rows with a byte >= 0x80 in the name, or without a legal word, are flagged
// and left to the host.  acc: hist [k], rows, tp, fp, fn over the rows scored here.
__global__ void __launch_bounds__(256)
eval_score_kernel(EvalTables T, const int32_t* __restrict__ ids, int n, int k, const long long* __restrict__ name_off,
                  const unsigned char* __restrict__ names, int32_t* __restrict__ rank_out, int32_t* __restrict__ first_out,
                  int32_t* __restrict__ flags_out, unsigned long long* __restrict__ acc) {
  const int lane = threadIdx.x & 31;
  for (long long row = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5; row < n; row += ((long long)gridDim.x * 256) >> 5) {
    const unsigned char* nm = names + name_off[row];
    const long long L = name_off[row + 1] - name_off[row];
    bool high = false, letters = false;
    int bars = 0;
    for (long long p = lane; p < L; p += 32) {
      const unsigned char c = nm[p];
      high |= c >= 0x80;
      letters |= ascii_letter(c);
      bars += c == '|';
    }
    high = __any_sync(kFull, high);
    letters = __any_sync(kFull, letters);
    bars = __reduce_add_sync(kFull, bars);
    int rank = -1, first = -1, legal_before = 0;
    if (!high) {
      for (int w = 0; w < k; w += 32) {
        const int i = w + lane;
        const int id = i < k ? ids[(long long)row * k + i] : -1;
        const bool lg = id >= 0 && id < T.Y && T.legal[id];
        const unsigned lm = __ballot_sync(kFull, lg);
        if (first < 0 && lm) first = __shfl_sync(kFull, id, __ffs(lm) - 1);
        const bool mt = lg && rank < 0 &&
                        norm_equal(nm, L, letters, T.norm + T.norm_off[id], T.norm_off[id + 1] - T.norm_off[id]);
        const unsigned mm = __ballot_sync(kFull, mt);
        if (rank < 0 && mm) rank = legal_before + __popc(lm & ((1u << (__ffs(mm) - 1)) - 1u));
        legal_before += __popc(lm);
      }
    }
    const int flags = (high ? 1 : 0) | (!high && first < 0 ? 2 : 0);
    if (lane == 0) {
      rank_out[row] = flags ? -1 : rank;
      first_out[row] = first;
      flags_out[row] = flags;
    }
    if (flags) continue;
    const unsigned char* g = T.words + T.word_off[first];
    const long long GL = T.word_off[first + 1] - T.word_off[first];
    int g_bars = 0;
    for (long long p = lane; p < GL; p += 32) g_bars += g[p] == '|';
    g_bars = __reduce_add_sync(kFull, g_bars);
    unsigned long long tp = 0, fp = 0, fn = 0;
    for (int j = lane; j <= g_bars; j += 32) {          // guess subtokens, with multiplicity
      long long s;
      const long long tl = subtoken(g, GL, j, &s);
      if (has_subtoken(nm, L, g + s, tl)) ++tp; else ++fp;
    }
    for (int j = lane; j <= bars; j += 32) {            // truth subtokens, with multiplicity
      long long s;
      const long long tl = subtoken(nm, L, j, &s);
      if (!has_subtoken(g, GL, nm + s, tl)) ++fn;
    }
    tp = __reduce_add_sync(kFull, (unsigned)tp);
    fp = __reduce_add_sync(kFull, (unsigned)fp);
    fn = __reduce_add_sync(kFull, (unsigned)fn);
    if (lane == 0) {
      if (rank >= 0) atomicAdd(acc + rank, 1ull);
      atomicAdd(acc + k, 1ull);
      atomicAdd(acc + k + 1, tp);
      atomicAdd(acc + k + 2, fp);
      atomicAdd(acc + k + 3, fn);
    }
  }
}

// ---- names Python's strict UTF-8 decoder accepts (c2v_reader_eval_check_utf8) ----------------------------------------
// Well-formed UTF-8 as str.decode("utf-8") takes it: no overlong forms, no surrogates (ED A0..BF), nothing above U+10FFFF.
__device__ bool utf8_valid(const unsigned char* s, long long n) {
  long long p = 0;
  while (p < n) {
    const unsigned char c = s[p];
    if (c < 0x80) { ++p; continue; }
    int len;
    unsigned char lo = 0x80, hi = 0xBF;                 // the range of the second byte
    if (c >= 0xC2 && c <= 0xDF) len = 2;
    else if (c >= 0xE0 && c <= 0xEF) { len = 3; if (c == 0xE0) lo = 0xA0; if (c == 0xED) hi = 0x9F; }
    else if (c >= 0xF0 && c <= 0xF4) { len = 4; if (c == 0xF0) lo = 0x90; if (c == 0xF4) hi = 0x8F; }
    else return false;
    if (p + len > n || s[p + 1] < lo || s[p + 1] > hi) return false;
    for (int i = 2; i < len; ++i)
      if (s[p + i] < 0x80 || s[p + i] > 0xBF) return false;
    p += len;
  }
  return true;
}

// *bad = the lowest queue row in [q0, q0 + n) whose name is not valid UTF-8 (left as is when there is none); one thread a row
__global__ void __launch_bounds__(256) eval_utf8_kernel(const long long* __restrict__ noff, const unsigned char* __restrict__ names,
                                                        long long q0, long long n, unsigned long long* __restrict__ bad) {
  for (long long j = (long long)blockIdx.x * 256 + threadIdx.x; j < n; j += (long long)gridDim.x * 256) {
    const long long o = noff[q0 + j];
    if (!utf8_valid(names + o, noff[q0 + j + 1] - o)) atomicMin(bad, (unsigned long long)(q0 + j));
  }
}

}  // namespace

struct c2v_reader {
  int device = 0, C = 0, num_sms = 1;
  DevVocab tok{}, pth{}, tgt{};
  // shuffle pool: rows [0, live) are the pool, [live, cap) room for the next chunk
  PoolRows pool{};
  long long pool_cap = 0, live = 0;
  // per-chunk scratch (sized for the largest chunk so far)
  long long text_cap = 0, row_cap = 0, pick_cap = 0;
  int *rec_cnt = nullptr, *nl_cnt = nullptr, *rec_base = nullptr, *nl_base = nullptr;     // [tiles + 1]
  long long *rec_off = nullptr, *rec_line = nullptr;                                        // [rows]
  uint8_t* keep = nullptr;                                                                  // [rows]
  int *keep_cnt = nullptr, *keep_base = nullptr;                                            // [row tiles + 1]
  int *holes = nullptr, *movers = nullptr;                                                  // [max(rows, picks)]
  long long* pick = nullptr;                                                                // [picks]
  uint8_t* tail = nullptr;                                                                  // [picks]
  unsigned long long* bad = nullptr;
  int* n_moves = nullptr;
  int* n_rec = nullptr;                                                                     // records of assembled shares
  // evaluation queue (c2v_reader_eval_*): rows [eq_head, eq_len) are queued in file order, row j's name is
  // eq_names[eq_noff[j], eq_noff[j + 1])
  PoolRows eq{};
  long long eq_cap = 0, eq_head = 0, eq_len = 0;
  long long* eq_noff = nullptr;                                                             // [eq_cap + 1]
  unsigned char* eq_names = nullptr;
  long long eq_names_cap = 0, eq_names_end = 0;
  long long eval_row_cap = 0;
  int *name_len = nullptr, *qlen = nullptr, *qoff = nullptr;                                // [eval rows (+ 1)]
  EvalTables tab{};                                                                         // c2v_reader_eval_tables
  unsigned char* tab_mem = nullptr;
  size_t tab_bytes = 0;
  long long oov_off = 0;                                                                    // the OOV word in tab.words
  int oov_len = 0;
  struct Status {
    int records, kept, newlines, name_bytes;
    unsigned long long bad;
    long long line, noff_head;
  } *host = nullptr;                                                                        // pinned read-back
  size_t bytes = 0;               // device memory held
};

namespace {

int rfail(int code, const std::string& msg) {
  c2v::set_global_error(msg);
  return code;
}

#define RD_CUDA(call)                                                                                   \
  do {                                                                                                  \
    cudaError_t _e = (call);                                                                            \
    if (_e != cudaSuccess) return rfail(C2V_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e)); \
  } while (0)

template <class T>
int realloc_dev(c2v_reader* r, T*& p, long long old_n, long long n) {
  if (p) { RD_CUDA(cudaFree(p)); r->bytes -= (size_t)old_n * sizeof(T); }
  p = nullptr;
  RD_CUDA(cudaMalloc(&p, (size_t)(n > 0 ? n : 1) * sizeof(T)));
  r->bytes += (size_t)n * sizeof(T);
  return C2V_OK;
}

// scratch for a chunk of `nbytes` bytes and up to `rows` records; draws of up to `picks` rows
int reserve_scratch(c2v_reader* r, long long nbytes, long long rows, long long picks, cudaStream_t st) {
  const long long tiles = (nbytes + kTile - 1) / kTile + 1, row_tiles = (rows + kRowTile - 1) / kRowTile + 1;
  const long long old_tiles = (r->text_cap + kTile - 1) / kTile + 1, old_row_tiles = (r->row_cap + kRowTile - 1) / kRowTile + 1;
  if (nbytes > r->text_cap || rows > r->row_cap || picks > r->pick_cap) RD_CUDA(cudaStreamSynchronize(st));
  int rc;
  if (nbytes > r->text_cap) {
    for (int** p : {&r->rec_cnt, &r->nl_cnt, &r->rec_base, &r->nl_base})
      if ((rc = realloc_dev(r, *p, r->text_cap ? old_tiles : 0, tiles))) return rc;
    r->text_cap = nbytes;
  }
  const long long old_idx = r->row_cap > r->pick_cap ? r->row_cap : r->pick_cap;     // holes / movers serve both
  const long long idx = rows > picks ? rows : picks;
  if (idx > old_idx) {
    if ((rc = realloc_dev(r, r->holes, old_idx, idx)) || (rc = realloc_dev(r, r->movers, old_idx, idx))) return rc;
  }
  if (rows > r->row_cap) {
    if ((rc = realloc_dev(r, r->rec_off, r->row_cap ? r->row_cap + 1 : 0, rows + 1)) ||
        (rc = realloc_dev(r, r->rec_line, r->row_cap ? r->row_cap + 1 : 0, rows + 1)) ||
        (rc = realloc_dev(r, r->keep, r->row_cap, rows)) ||
        (rc = realloc_dev(r, r->keep_cnt, r->row_cap ? old_row_tiles : 0, row_tiles)) ||
        (rc = realloc_dev(r, r->keep_base, r->row_cap ? old_row_tiles : 0, row_tiles)))
      return rc;
    r->row_cap = rows;
  }
  if (picks > r->pick_cap) {
    if ((rc = realloc_dev(r, r->pick, r->pick_cap, picks)) || (rc = realloc_dev(r, r->tail, r->pick_cap, picks))) return rc;
    r->pick_cap = picks;
  }
  return C2V_OK;
}

// room for `more` rows behind the live end; the live rows move to the grown arrays
int reserve_pool(c2v_reader* r, long long more, cudaStream_t st) {
  const long long need = r->live + more;
  if (need <= r->pool_cap) return C2V_OK;
  long long cap = r->pool_cap ? 2 * r->pool_cap : 1024;
  if (cap < need) cap = need;
  const size_t C = (size_t)r->C, n = (size_t)r->live;
  PoolRows g{};
  RD_CUDA(cudaMalloc(&g.src, (size_t)cap * C * 4));
  RD_CUDA(cudaMalloc(&g.path, (size_t)cap * C * 4));
  RD_CUDA(cudaMalloc(&g.dst, (size_t)cap * C * 4));
  RD_CUDA(cudaMalloc(&g.mask, (size_t)cap * C * 4));
  RD_CUDA(cudaMalloc(&g.target, (size_t)cap * 4));
  if (r->pool_cap) {
    RD_CUDA(cudaMemcpyAsync(g.src, r->pool.src, n * C * 4, cudaMemcpyDeviceToDevice, st));
    RD_CUDA(cudaMemcpyAsync(g.path, r->pool.path, n * C * 4, cudaMemcpyDeviceToDevice, st));
    RD_CUDA(cudaMemcpyAsync(g.dst, r->pool.dst, n * C * 4, cudaMemcpyDeviceToDevice, st));
    RD_CUDA(cudaMemcpyAsync(g.mask, r->pool.mask, n * C * 4, cudaMemcpyDeviceToDevice, st));
    RD_CUDA(cudaMemcpyAsync(g.target, r->pool.target, n * 4, cudaMemcpyDeviceToDevice, st));
    RD_CUDA(cudaStreamSynchronize(st));
    for (void* p : {(void*)r->pool.src, (void*)r->pool.path, (void*)r->pool.dst, (void*)r->pool.mask, (void*)r->pool.target})
      RD_CUDA(cudaFree(p));
    r->bytes -= (size_t)r->pool_cap * (4 * C + 1) * 4;
  }
  r->pool = g;
  r->pool_cap = cap;
  r->bytes += (size_t)cap * (4 * C + 1) * 4;
  return C2V_OK;
}

// evaluate-mode scratch for chunks of up to `rows` records
int reserve_eval(c2v_reader* r, long long rows, cudaStream_t st) {
  if (rows <= r->eval_row_cap) return C2V_OK;
  RD_CUDA(cudaStreamSynchronize(st));
  const long long old = r->eval_row_cap;
  int rc;
  if ((rc = realloc_dev(r, r->name_len, old, rows)) || (rc = realloc_dev(r, r->qlen, old, rows)) ||
      (rc = realloc_dev(r, r->qoff, old ? old + 1 : 0, rows + 1)))
    return rc;
  r->eval_row_cap = rows;
  return C2V_OK;
}

// room in the evaluation queue for `rows` rows from row 0 and `name_bytes` name bytes; the queued content moves along
int reserve_queue(c2v_reader* r, long long rows, long long name_bytes, cudaStream_t st) {
  const size_t C = (size_t)r->C, n = (size_t)r->eq_len;
  if (rows > r->eq_cap) {
    long long cap = r->eq_cap ? 2 * r->eq_cap : 1024;
    if (cap < rows) cap = rows;
    PoolRows g{};
    long long* noff = nullptr;
    RD_CUDA(cudaMalloc(&g.src, (size_t)cap * C * 4));
    RD_CUDA(cudaMalloc(&g.path, (size_t)cap * C * 4));
    RD_CUDA(cudaMalloc(&g.dst, (size_t)cap * C * 4));
    RD_CUDA(cudaMalloc(&g.mask, (size_t)cap * C * 4));
    RD_CUDA(cudaMalloc(&g.target, (size_t)cap * 4));
    RD_CUDA(cudaMalloc(&noff, (size_t)(cap + 1) * 8));
    if (r->eq_cap) {
      RD_CUDA(cudaMemcpyAsync(g.src, r->eq.src, n * C * 4, cudaMemcpyDeviceToDevice, st));
      RD_CUDA(cudaMemcpyAsync(g.path, r->eq.path, n * C * 4, cudaMemcpyDeviceToDevice, st));
      RD_CUDA(cudaMemcpyAsync(g.dst, r->eq.dst, n * C * 4, cudaMemcpyDeviceToDevice, st));
      RD_CUDA(cudaMemcpyAsync(g.mask, r->eq.mask, n * C * 4, cudaMemcpyDeviceToDevice, st));
      RD_CUDA(cudaMemcpyAsync(g.target, r->eq.target, n * 4, cudaMemcpyDeviceToDevice, st));
      RD_CUDA(cudaMemcpyAsync(noff, r->eq_noff, (n + 1) * 8, cudaMemcpyDeviceToDevice, st));
      RD_CUDA(cudaStreamSynchronize(st));
      for (void* p : {(void*)r->eq.src, (void*)r->eq.path, (void*)r->eq.dst, (void*)r->eq.mask, (void*)r->eq.target,
                      (void*)r->eq_noff})
        RD_CUDA(cudaFree(p));
      r->bytes -= (size_t)r->eq_cap * (4 * C + 1) * 4 + (size_t)(r->eq_cap + 1) * 8;
    }
    r->eq = g;
    r->eq_noff = noff;
    r->eq_cap = cap;
    r->bytes += (size_t)cap * (4 * C + 1) * 4 + (size_t)(cap + 1) * 8;
  }
  if (name_bytes > r->eq_names_cap) {
    long long cap = r->eq_names_cap ? 2 * r->eq_names_cap : 1 << 16;
    if (cap < name_bytes) cap = name_bytes;
    unsigned char* g = nullptr;
    RD_CUDA(cudaMalloc(&g, (size_t)cap));
    if (r->eq_names) {
      RD_CUDA(cudaMemcpyAsync(g, r->eq_names, (size_t)r->eq_names_end, cudaMemcpyDeviceToDevice, st));
      RD_CUDA(cudaStreamSynchronize(st));
      RD_CUDA(cudaFree(r->eq_names));
      r->bytes -= (size_t)r->eq_names_cap;
    }
    r->eq_names = g;
    r->eq_names_cap = cap;
    r->bytes += (size_t)cap;
  }
  return C2V_OK;
}

int row_grid(const c2v_reader* r, long long rows) {            // one warp per row, 8 rows a block
  long long g = (rows + 7) / 8;
  if (g > (long long)r->num_sms * 8) g = (long long)r->num_sms * 8;
  return (int)(g > 0 ? g : 1);
}

DevVocab dev_vocab(const c2v_reader_vocab& v) {
  return DevVocab{(const DevSlot*)v.slots, (const unsigned char*)v.bytes, (unsigned long long)v.mask, v.oov, v.pad};
}

size_t parse_smem(int C) { return (size_t)kParseWarps * 3 * C * sizeof(longlong2); }

// line index and parse of text[0, nbytes) (nbytes > 0, `tiles` tiles of it, scratch reserved for `cap` records): the
// first `cap` records land in rows[0, cap) and keep[0, cap), the lowest malformed one in r->bad
int index_and_parse(c2v_reader* r, const unsigned char* t, long long nbytes, int tiles, long long cap, PoolRows rows,
                    uint8_t* keep, cudaStream_t st, int mode = 0, int* name_len = nullptr) {
  RD_CUDA(cudaMemsetAsync(r->bad, 0xff, sizeof(unsigned long long), st));
  line_count_kernel<<<tiles, kTileThreads, 0, st>>>(t, nbytes, r->rec_cnt, r->nl_cnt);
  exclusive_scan_kernel<<<1, 1024, 0, st>>>(r->rec_cnt, r->rec_base, tiles);
  exclusive_scan_kernel<<<1, 1024, 0, st>>>(r->nl_cnt, r->nl_base, tiles);
  line_index_kernel<<<tiles, kTileThreads, 0, st>>>(t, nbytes, r->rec_base, r->nl_base, cap, r->rec_off, r->rec_line);
  ParseArgs a{t, nbytes, r->C, r->tok, r->pth, r->tgt, r->rec_off, r->rec_base + tiles, cap,
              rows.src, rows.path, rows.dst, rows.target, rows.mask, keep, r->bad, mode, name_len};
  long long grid = (cap + kParseWarps - 1) / kParseWarps;
  if (grid > (long long)r->num_sms * 16) grid = (long long)r->num_sms * 16;
  parse_kernel<<<(unsigned)grid, 32 * kParseWarps, parse_smem(r->C), st>>>(a);
  RD_CUDA(cudaGetLastError());
  return C2V_OK;
}

// keep_count + scan + commit_index + move_rows over the `cap`-bounded records (*n_rec) just behind the live end, then
// reads the kept count back (synchronises st) and advances the live end.  The records' keep flags are in r->keep.
int commit_records(c2v_reader* r, const int* n_rec, long long cap, int64_t* kept, cudaStream_t st) {
  const int row_tiles = (int)((cap + kRowTile - 1) / kRowTile);
  keep_count_kernel<<<row_tiles, 256, 0, st>>>(r->keep, n_rec, cap, r->keep_cnt);
  exclusive_scan_kernel<<<1, 1024, 0, st>>>(r->keep_cnt, r->keep_base, row_tiles);
  commit_index_kernel<<<row_tiles, 256, 0, st>>>(r->keep, n_rec, cap, r->keep_base, row_tiles, r->holes, r->movers,
                                                 r->n_moves);
  move_rows_kernel<<<r->num_sms * 8, 256, 0, st>>>(r->pool, r->C, r->live, r->holes, r->movers, r->n_moves);
  RD_CUDA(cudaGetLastError());
  RD_CUDA(cudaMemcpyAsync(&r->host->kept, r->keep_base + row_tiles, sizeof(int), cudaMemcpyDeviceToHost, st));
  RD_CUDA(cudaStreamSynchronize(st));
  *kept = r->host->kept;
  r->live += r->host->kept;
  return C2V_OK;
}

}  // namespace

extern "C" {

int c2v_reader_create(int32_t max_contexts, const c2v_reader_vocab* tok, const c2v_reader_vocab* path,
                      const c2v_reader_vocab* target, int device, c2v_reader** out) {
  if (!out || !tok || !path || !target) return rfail(C2V_ERR_INVALID, "c2v_reader_create: NULL argument");
  *out = nullptr;
  if (max_contexts < 1) return rfail(C2V_ERR_INVALID, "c2v_reader_create: max_contexts must be >= 1");
  for (const c2v_reader_vocab* v : {tok, path, target})
    if (!v->slots || !v->bytes || ((v->mask + 1) & v->mask) != 0)
      return rfail(C2V_ERR_INVALID, "c2v_reader_create: a vocabulary needs device slots, bytes and a 2^k - 1 mask");
  RD_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  RD_CUDA(cudaGetDeviceProperties(&prop, device));
  if (parse_smem(max_contexts) > prop.sharedMemPerBlockOptin)
    return rfail(C2V_ERR_UNSUPPORTED, "c2v_reader_create: max_contexts too large for the parse kernel's shared memory");
  RD_CUDA(cudaFuncSetAttribute(parse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)parse_smem(max_contexts)));
  c2v_reader* r = new c2v_reader();
  r->device = device;
  r->C = max_contexts;
  r->num_sms = prop.multiProcessorCount;
  r->tok = dev_vocab(*tok);
  r->pth = dev_vocab(*path);
  r->tgt = dev_vocab(*target);
  cudaError_t e = cudaMalloc(&r->bad, sizeof(unsigned long long));
  if (e == cudaSuccess) e = cudaMalloc(&r->n_moves, sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&r->n_rec, sizeof(int));
  if (e == cudaSuccess) e = cudaHostAlloc((void**)&r->host, sizeof(c2v_reader::Status), cudaHostAllocDefault);
  if (e != cudaSuccess) {
    c2v_reader_destroy(r);
    return rfail(C2V_ERR_CUDA, std::string("c2v_reader_create: ") + cudaGetErrorString(e));
  }
  r->bytes = sizeof(unsigned long long) + 2 * sizeof(int);
  *out = r;
  return C2V_OK;
}

void c2v_reader_destroy(c2v_reader* r) {
  if (!r) return;
  cudaSetDevice(r->device);
  cudaDeviceSynchronize();
  for (void* p : {(void*)r->pool.src, (void*)r->pool.path, (void*)r->pool.dst, (void*)r->pool.mask, (void*)r->pool.target,
                  (void*)r->rec_cnt, (void*)r->nl_cnt, (void*)r->rec_base, (void*)r->nl_base, (void*)r->rec_off,
                  (void*)r->rec_line, (void*)r->keep, (void*)r->keep_cnt, (void*)r->keep_base, (void*)r->holes,
                  (void*)r->movers, (void*)r->pick, (void*)r->tail, (void*)r->bad, (void*)r->n_moves, (void*)r->n_rec,
                  (void*)r->eq.src, (void*)r->eq.path, (void*)r->eq.dst, (void*)r->eq.mask, (void*)r->eq.target,
                  (void*)r->eq_noff, (void*)r->eq_names, (void*)r->name_len, (void*)r->qlen, (void*)r->qoff,
                  (void*)r->tab_mem})
    if (p) cudaFree(p);
  if (r->host) cudaFreeHost(r->host);
  delete r;
}

int c2v_reader_parse_chunk(c2v_reader* r, const char* text, int64_t nbytes, int64_t* kept, int64_t* bad_line,
                           int32_t* bad_kind, void* stream) {
  if (!r || !text || !kept || !bad_line || !bad_kind || nbytes < 0)
    return rfail(C2V_ERR_INVALID, "c2v_reader_parse_chunk: NULL argument or negative size");
  *kept = 0; *bad_line = -1; *bad_kind = 0;
  if (nbytes == 0) return C2V_OK;
  RD_CUDA(cudaSetDevice(r->device));
  cudaStream_t st = (cudaStream_t)stream;
  const long long cap = nbytes / (r->C + 1) + 1;      // a well-formed line is at least MAX_CONTEXTS spaces + a newline long
  int rc;
  if ((rc = reserve_scratch(r, nbytes, cap, 0, st)) || (rc = reserve_pool(r, cap, st))) return rc;
  const int tiles = (int)((nbytes + kTile - 1) / kTile), row_tiles = (int)((cap + kRowTile - 1) / kRowTile);
  const unsigned char* t = (const unsigned char*)text;
  const long long l0 = r->live * r->C;
  const PoolRows tail{r->pool.src + l0, r->pool.path + l0, r->pool.dst + l0, r->pool.target + r->live, r->pool.mask + l0};
  if ((rc = index_and_parse(r, t, nbytes, tiles, cap, tail, r->keep, st))) return rc;
  keep_count_kernel<<<row_tiles, 256, 0, st>>>(r->keep, r->rec_base + tiles, cap, r->keep_cnt);
  exclusive_scan_kernel<<<1, 1024, 0, st>>>(r->keep_cnt, r->keep_base, row_tiles);
  commit_index_kernel<<<row_tiles, 256, 0, st>>>(r->keep, r->rec_base + tiles, cap, r->keep_base, row_tiles, r->holes,
                                                 r->movers, r->n_moves);
  move_rows_kernel<<<r->num_sms * 8, 256, 0, st>>>(r->pool, r->C, r->live, r->holes, r->movers, r->n_moves);
  RD_CUDA(cudaGetLastError());
  RD_CUDA(cudaMemcpyAsync(&r->host->records, r->rec_base + tiles, sizeof(int), cudaMemcpyDeviceToHost, st));
  RD_CUDA(cudaMemcpyAsync(&r->host->kept, r->keep_base + row_tiles, sizeof(int), cudaMemcpyDeviceToHost, st));
  RD_CUDA(cudaMemcpyAsync(&r->host->bad, r->bad, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  RD_CUDA(cudaStreamSynchronize(st));
  if (r->host->records > cap) {
    *bad_kind = 3;
    return rfail(C2V_ERR_INVALID, "c2v_reader_parse_chunk: more records than a chunk of this size holds well-formed lines");
  }
  if (r->host->bad != ~0ull) {
    const long long li = (long long)(r->host->bad >> 2);
    RD_CUDA(cudaMemcpyAsync(&r->host->line, r->rec_line + li, sizeof(long long), cudaMemcpyDeviceToHost, st));
    RD_CUDA(cudaStreamSynchronize(st));
    *bad_line = r->host->line;
    *bad_kind = (int32_t)(r->host->bad & 3);
    return rfail(C2V_ERR_INVALID, std::string("c2v_reader_parse_chunk: malformed line ") + std::to_string(*bad_line) +
                                      (*bad_kind == 2 ? " (a context has more than 3 parts)" : " (field count)"));
  }
  *kept = r->host->kept;
  r->live += r->host->kept;
  return C2V_OK;
}

int c2v_reader_draw(c2v_reader* r, const int64_t* pick, int32_t b, int32_t lo, int32_t hi, int32_t* src, int32_t* path,
                    int32_t* tgt, float* mask, int32_t* target, void* stream) {
  if (!r || !pick) return rfail(C2V_ERR_INVALID, "c2v_reader_draw: NULL argument");
  if (b < 1 || b > r->live) return rfail(C2V_ERR_INVALID, "c2v_reader_draw: b must be in [1, live rows]");
  if (lo < 0 || lo > hi || hi > b) return rfail(C2V_ERR_INVALID, "c2v_reader_draw: need 0 <= lo <= hi <= b");
  if (hi > lo && (!src || !path || !tgt || !mask || !target)) return rfail(C2V_ERR_INVALID, "c2v_reader_draw: NULL output");
  RD_CUDA(cudaSetDevice(r->device));
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if ((rc = reserve_scratch(r, 0, 0, b, st))) return rc;
  RD_CUDA(cudaMemcpyAsync(r->pick, pick, (size_t)b * sizeof(long long), cudaMemcpyHostToDevice, st));
  draw_index_kernel<<<1, 1024, 0, st>>>(r->pick, b, r->live, r->tail, r->holes, r->movers, r->n_moves);
  if (hi > lo) {
    long long grid = ((long long)(hi - lo) * 32 + 255) / 256;
    if (grid > (long long)r->num_sms * 8) grid = (long long)r->num_sms * 8;
    gather_kernel<<<(unsigned)grid, 256, 0, st>>>(r->pool, r->C, r->pick, lo, hi, PoolRows{src, path, tgt, target, mask});
  }
  // every picked row has been gathered (same stream) before a hole is overwritten
  move_rows_kernel<<<r->num_sms * 4, 256, 0, st>>>(r->pool, r->C, 0, r->holes, r->movers, r->n_moves);
  RD_CUDA(cudaGetLastError());
  r->live -= b;
  return C2V_OK;
}

size_t c2v_reader_stage_bytes(int32_t max_contexts, int64_t rows) {
  if (max_contexts < 1 || rows < 1) return 0;
  return (size_t)stage_layout(max_contexts, rows).bytes;
}

int c2v_reader_parse_share(c2v_reader* r, const char* text, int64_t nbytes, int64_t chunk_bytes, void* stage,
                           int64_t stage_rows, c2v_reader_share_status* status, void* stream) {
  if (!r || !stage || !status || (nbytes > 0 && !text))
    return rfail(C2V_ERR_INVALID, "c2v_reader_parse_share: NULL argument");
  if (nbytes < 0 || chunk_bytes < nbytes || stage_rows < 1)
    return rfail(C2V_ERR_INVALID, "c2v_reader_parse_share: need 0 <= nbytes <= chunk_bytes and stage_rows >= 1");
  RD_CUDA(cudaSetDevice(r->device));
  cudaStream_t st = (cudaStream_t)stream;
  c2v_reader_share_status s{};
  s.rows = stage_rows;
  s.bad_line = -1;
  if (nbytes > 0) {
    const unsigned char* t = (const unsigned char*)text;
    unsigned char* g = (unsigned char*)stage;
    const StageLayout L = stage_layout(r->C, stage_rows);
    const PoolRows rows{(int32_t*)(g + L.src), (int32_t*)(g + L.path), (int32_t*)(g + L.dst), (int32_t*)(g + L.target),
                        (float*)(g + L.mask)};
    const int tiles = (int)((nbytes + kTile - 1) / kTile), row_tiles = (int)((stage_rows + kRowTile - 1) / kRowTile);
    int rc;
    if ((rc = reserve_scratch(r, nbytes, stage_rows, 0, st))) return rc;
    if ((rc = index_and_parse(r, t, nbytes, tiles, stage_rows, rows, g + L.keep, st))) return rc;
    keep_count_kernel<<<row_tiles, 256, 0, st>>>(g + L.keep, r->rec_base + tiles, stage_rows, r->keep_cnt);
    exclusive_scan_kernel<<<1, 1024, 0, st>>>(r->keep_cnt, r->keep_base, row_tiles);
    RD_CUDA(cudaGetLastError());
    RD_CUDA(cudaMemcpyAsync(&r->host->records, r->rec_base + tiles, sizeof(int), cudaMemcpyDeviceToHost, st));
    RD_CUDA(cudaMemcpyAsync(&r->host->newlines, r->nl_base + tiles, sizeof(int), cudaMemcpyDeviceToHost, st));
    RD_CUDA(cudaMemcpyAsync(&r->host->kept, r->keep_base + row_tiles, sizeof(int), cudaMemcpyDeviceToHost, st));
    RD_CUDA(cudaMemcpyAsync(&r->host->bad, r->bad, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    RD_CUDA(cudaStreamSynchronize(st));
    s.records = r->host->records;
    s.newlines = r->host->newlines;
    if (s.records > stage_rows) {
      // more records than the share holds well-formed lines: one of them is malformed.  The first pass's last record ran
      // to the end of the text, so its verdict is void; the lowest malformed line is found in a second pass over every
      // record, in the pool's room behind its live end.  With more records than the whole chunk holds well-formed lines
      // the chunk fails with kind 3 whatever the lines are, and no pass is needed.
      s.overflow = 1;
      r->host->bad = ~0ull;
      const long long chunk_cap = chunk_bytes / (r->C + 1) + 1;
      if (s.records <= chunk_cap) {
        if ((rc = reserve_scratch(r, nbytes, s.records, 0, st)) || (rc = reserve_pool(r, s.records, st))) return rc;
        const long long l0 = r->live * r->C;
        const PoolRows tail{r->pool.src + l0, r->pool.path + l0, r->pool.dst + l0, r->pool.target + r->live,
                            r->pool.mask + l0};
        if ((rc = index_and_parse(r, t, nbytes, tiles, s.records, tail, r->keep, st))) return rc;
        RD_CUDA(cudaMemcpyAsync(&r->host->bad, r->bad, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
        RD_CUDA(cudaStreamSynchronize(st));
      }
    }
    if (r->host->bad != ~0ull) {
      const long long li = (long long)(r->host->bad >> 2);
      RD_CUDA(cudaMemcpyAsync(&r->host->line, r->rec_line + li, sizeof(long long), cudaMemcpyDeviceToHost, st));
      RD_CUDA(cudaStreamSynchronize(st));
      s.bad_line = r->host->line;
      s.bad_kind = (int32_t)(r->host->bad & 3);
    } else if (!s.overflow) {
      s.kept = r->host->kept;
    }
  }
  RD_CUDA(cudaMemcpyAsync(stage, &s, sizeof(s), cudaMemcpyHostToDevice, st));
  RD_CUDA(cudaStreamSynchronize(st));
  *status = s;
  return C2V_OK;
}

int c2v_reader_commit_shares(c2v_reader* r, const void* const* stages, const int64_t* records, int32_t n_shares,
                             int64_t* kept, void* stream) {
  if (!r || !stages || !records || !kept) return rfail(C2V_ERR_INVALID, "c2v_reader_commit_shares: NULL argument");
  if (n_shares < 1 || n_shares > kMaxShares)
    return rfail(C2V_ERR_INVALID, "c2v_reader_commit_shares: n_shares must be in [1, " + std::to_string(kMaxShares) + "]");
  *kept = 0;
  AssembleArgs a{};
  long long total = 0;
  for (int i = 0; i < n_shares; ++i) {
    if (records[i] < 0 || (records[i] > 0 && !stages[i]))
      return rfail(C2V_ERR_INVALID, "c2v_reader_commit_shares: a share with records needs its stage");
    a.share[i] = ShareSrc{(const unsigned char*)stages[i], total, (long long)records[i]};
    total += records[i];
  }
  if (total == 0) return C2V_OK;
  if (total > INT32_MAX) return rfail(C2V_ERR_INVALID, "c2v_reader_commit_shares: more than 2^31 - 1 records");
  RD_CUDA(cudaSetDevice(r->device));
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if ((rc = reserve_scratch(r, 0, total, 0, st)) || (rc = reserve_pool(r, total, st))) return rc;
  a.n = n_shares;
  a.C = r->C;
  a.pool = r->pool;
  a.live = r->live;
  a.keep = r->keep;
  a.n_rec = r->n_rec;
  a.total = total;
  const int per = (r->num_sms * 4 + n_shares - 1) / n_shares;
  assemble_shares_kernel<<<dim3((unsigned)per, (unsigned)n_shares), 256, 0, st>>>(a);
  RD_CUDA(cudaGetLastError());
  return commit_records(r, r->n_rec, total, kept, st);
}


int c2v_reader_eval_tables(c2v_reader* r, int32_t n_words, const char* words, const int64_t* word_off, const char* norm,
                           const int64_t* norm_off, const uint8_t* legal, void* stream) {
  if (!r || !word_off || !norm_off || !legal || (word_off[n_words > 0 ? n_words : 0] > 0 && !words))
    return rfail(C2V_ERR_INVALID, "c2v_reader_eval_tables: NULL argument");
  if (n_words <= r->tgt.oov || r->tgt.oov < 0)
    return rfail(C2V_ERR_INVALID, "c2v_reader_eval_tables: the tables must cover every target word, the OOV word included");
  if (word_off[0] != 0 || norm_off[0] != 0) return rfail(C2V_ERR_INVALID, "c2v_reader_eval_tables: offsets start at 0");
  for (int i = 0; i < n_words; ++i)
    if (word_off[i + 1] < word_off[i] || norm_off[i + 1] < norm_off[i])
      return rfail(C2V_ERR_INVALID, "c2v_reader_eval_tables: offsets must not decrease");
  RD_CUDA(cudaSetDevice(r->device));
  cudaStream_t st = (cudaStream_t)stream;
  const long long Y = n_words, wb = word_off[Y], nb = norm_off[Y];
  const long long o_woff = 0, o_noff = align256(o_woff + (Y + 1) * 8), o_legal = align256(o_noff + (Y + 1) * 8),
                  o_words = align256(o_legal + Y), o_norm = align256(o_words + wb), total = align256(o_norm + nb);
  RD_CUDA(cudaStreamSynchronize(st));
  if (r->tab_mem) {
    RD_CUDA(cudaFree(r->tab_mem));
    r->bytes -= r->tab_bytes;
    r->tab_mem = nullptr;
    r->tab = EvalTables{};
  }
  RD_CUDA(cudaMalloc(&r->tab_mem, (size_t)total));
  r->tab_bytes = (size_t)total;
  r->bytes += r->tab_bytes;
  unsigned char* m = r->tab_mem;
  RD_CUDA(cudaMemcpyAsync(m + o_woff, word_off, (size_t)(Y + 1) * 8, cudaMemcpyHostToDevice, st));
  RD_CUDA(cudaMemcpyAsync(m + o_noff, norm_off, (size_t)(Y + 1) * 8, cudaMemcpyHostToDevice, st));
  RD_CUDA(cudaMemcpyAsync(m + o_legal, legal, (size_t)Y, cudaMemcpyHostToDevice, st));
  if (wb) RD_CUDA(cudaMemcpyAsync(m + o_words, words, (size_t)wb, cudaMemcpyHostToDevice, st));
  if (nb) RD_CUDA(cudaMemcpyAsync(m + o_norm, norm, (size_t)nb, cudaMemcpyHostToDevice, st));
  RD_CUDA(cudaStreamSynchronize(st));
  r->tab = EvalTables{m + o_words, (const long long*)(m + o_woff), m + o_norm, (const long long*)(m + o_noff),
                      m + o_legal, (int)Y};
  r->oov_off = word_off[r->tgt.oov];
  r->oov_len = (int)(word_off[r->tgt.oov + 1] - word_off[r->tgt.oov]);
  return C2V_OK;
}

int c2v_reader_eval_append(c2v_reader* r, const char* text, int64_t nbytes, int64_t* appended, int64_t* name_bytes,
                           int64_t* bad_line, int32_t* bad_kind, void* stream) {
  if (!r || !text || !appended || !name_bytes || !bad_line || !bad_kind || nbytes < 0)
    return rfail(C2V_ERR_INVALID, "c2v_reader_eval_append: NULL argument or negative size");
  *appended = 0; *bad_line = -1; *bad_kind = 0;
  *name_bytes = r->eq_names_end;
  if (!r->tab_mem) return rfail(C2V_ERR_STATE, "c2v_reader_eval_append: upload the tables first (c2v_reader_eval_tables)");
  if (nbytes == 0) return C2V_OK;
  RD_CUDA(cudaSetDevice(r->device));
  cudaStream_t st = (cudaStream_t)stream;
  const long long cap = nbytes / (r->C + 1) + 1;      // a well-formed line is at least MAX_CONTEXTS spaces + a newline long
  int rc;
  if ((rc = reserve_scratch(r, nbytes, cap, 0, st)) || (rc = reserve_pool(r, cap, st)) || (rc = reserve_eval(r, cap, st)))
    return rc;
  const int tiles = (int)((nbytes + kTile - 1) / kTile), row_tiles = (int)((cap + kRowTile - 1) / kRowTile);
  const unsigned char* t = (const unsigned char*)text;
  const long long l0 = r->live * r->C;
  const PoolRows room{r->pool.src + l0, r->pool.path + l0, r->pool.dst + l0, r->pool.target + r->live, r->pool.mask + l0};
  if ((rc = index_and_parse(r, t, nbytes, tiles, cap, room, r->keep, st, 1, r->name_len))) return rc;
  const int* n_rec = r->rec_base + tiles;
  keep_count_kernel<<<row_tiles, 256, 0, st>>>(r->keep, n_rec, cap, r->keep_cnt);
  exclusive_scan_kernel<<<1, 1024, 0, st>>>(r->keep_cnt, r->keep_base, row_tiles);
  eval_index_kernel<<<row_tiles, 256, 0, st>>>(r->keep, n_rec, cap, r->keep_base, row_tiles, r->name_len, r->oov_len,
                                               r->movers, r->qlen);
  exclusive_scan_kernel<<<1, 1024, 0, st>>>(r->qlen, r->qoff, (int)cap);
  RD_CUDA(cudaGetLastError());
  RD_CUDA(cudaMemcpyAsync(&r->host->records, n_rec, sizeof(int), cudaMemcpyDeviceToHost, st));
  RD_CUDA(cudaMemcpyAsync(&r->host->kept, r->keep_base + row_tiles, sizeof(int), cudaMemcpyDeviceToHost, st));
  RD_CUDA(cudaMemcpyAsync(&r->host->name_bytes, r->qoff + cap, sizeof(int), cudaMemcpyDeviceToHost, st));
  RD_CUDA(cudaMemcpyAsync(&r->host->bad, r->bad, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  if (r->eq_len > r->eq_head)
    RD_CUDA(cudaMemcpyAsync(&r->host->noff_head, r->eq_noff + r->eq_head, sizeof(long long), cudaMemcpyDeviceToHost, st));
  RD_CUDA(cudaStreamSynchronize(st));
  if (r->host->records > cap) {
    *bad_kind = 3;
    return rfail(C2V_ERR_INVALID, "c2v_reader_eval_append: more records than a chunk of this size holds well-formed lines");
  }
  if (r->host->bad != ~0ull) {
    const long long li = (long long)(r->host->bad >> 2);
    RD_CUDA(cudaMemcpyAsync(&r->host->line, r->rec_line + li, sizeof(long long), cudaMemcpyDeviceToHost, st));
    RD_CUDA(cudaStreamSynchronize(st));
    *bad_line = r->host->line;
    *bad_kind = (int32_t)(r->host->bad & 3);
    return rfail(C2V_ERR_INVALID, std::string("c2v_reader_eval_append: malformed line ") + std::to_string(*bad_line) +
                                      (*bad_kind == 2 ? " (a context has more than 3 parts)" : " (field count)"));
  }
  // the rows taken so far leave the queue: the rest moves to its front when the two ranges do not overlap
  const long long left = r->eq_len - r->eq_head;
  if (left == 0) {
    r->eq_head = r->eq_len = r->eq_names_end = 0;
  } else if (r->eq_head > 0 && left < r->eq_head && r->eq_names_end - r->host->noff_head <= r->host->noff_head) {
    eval_compact_kernel<<<row_grid(r, left), 256, 0, st>>>(r->eq, r->C, r->eq_head, left, r->eq_noff, r->eq_names);
    RD_CUDA(cudaGetLastError());
    r->eq_names_end -= r->host->noff_head;
    r->eq_head = 0;
    r->eq_len = left;
  }
  const int kept = r->host->kept;
  const long long nb = r->host->name_bytes;
  if (kept > 0) {
    if ((rc = reserve_queue(r, r->eq_len + kept, r->eq_names_end + nb, st))) return rc;
    const long long q0 = r->eq_len * r->C;
    EvalAppendArgs a{room, PoolRows{r->eq.src + q0, r->eq.path + q0, r->eq.dst + q0, r->eq.target + r->eq_len,
                                    r->eq.mask + q0},
                     r->C, kept, r->movers, r->qoff, r->rec_off, r->name_len, t, r->tab.words + r->oov_off, r->oov_len,
                     r->eq_names_end, r->eq_names, r->eq_noff + r->eq_len, nb};
    eval_append_kernel<<<row_grid(r, kept), 256, 0, st>>>(a);
    RD_CUDA(cudaGetLastError());
    r->eq_len += kept;
    r->eq_names_end += nb;
  }
  *appended = kept;
  *name_bytes = r->eq_names_end;
  return C2V_OK;
}

int c2v_reader_eval_take(c2v_reader* r, int32_t b, int32_t* src, int32_t* path, int32_t* tgt, float* mask,
                         int32_t* target, int64_t* name_off, char* names, int64_t names_cap, void* stream) {
  if (!r || !src || !path || !tgt || !mask || !target || !name_off || !names)
    return rfail(C2V_ERR_INVALID, "c2v_reader_eval_take: NULL argument");
  if (b < 1 || b > r->eq_len - r->eq_head)
    return rfail(C2V_ERR_INVALID, "c2v_reader_eval_take: b must be in [1, queued rows]");
  if (names_cap < r->eq_names_end)
    return rfail(C2V_ERR_INVALID, "c2v_reader_eval_take: names_cap must be at least the name bytes the last append reported");
  RD_CUDA(cudaSetDevice(r->device));
  cudaStream_t st = (cudaStream_t)stream;
  eval_take_kernel<<<row_grid(r, b), 256, 0, st>>>(r->eq, r->C, r->eq_head, b, r->eq_noff, r->eq_names,
                                                   PoolRows{src, path, tgt, target, mask}, (long long*)name_off,
                                                   (unsigned char*)names, names_cap);
  RD_CUDA(cudaGetLastError());
  r->eq_head += b;
  return C2V_OK;
}

int64_t c2v_reader_eval_queued(const c2v_reader* r) { return r ? r->eq_len - r->eq_head : -1; }

int c2v_reader_eval_check_utf8(c2v_reader* r, int64_t rows, char* name, int64_t name_cap, int64_t* name_len, void* stream) {
  if (!r || !name_len || rows < 0 || name_cap < 0 || (name_cap && !name))
    return rfail(C2V_ERR_INVALID, "c2v_reader_eval_check_utf8: NULL argument or negative size");
  if (rows > r->eq_len - r->eq_head)
    return rfail(C2V_ERR_INVALID, "c2v_reader_eval_check_utf8: rows must be at most the queued rows");
  *name_len = -1;
  if (rows == 0) return C2V_OK;
  RD_CUDA(cudaSetDevice(r->device));
  cudaStream_t st = (cudaStream_t)stream;
  const long long q0 = r->eq_len - rows;
  RD_CUDA(cudaMemsetAsync(r->bad, 0xff, sizeof(unsigned long long), st));
  eval_utf8_kernel<<<row_grid(r, rows), 256, 0, st>>>(r->eq_noff, r->eq_names, q0, rows, r->bad);
  RD_CUDA(cudaGetLastError());
  RD_CUDA(cudaMemcpyAsync(&r->host->bad, r->bad, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  RD_CUDA(cudaStreamSynchronize(st));
  if (r->host->bad == ~0ull) return C2V_OK;
  long long off[2];
  RD_CUDA(cudaMemcpyAsync(off, r->eq_noff + r->host->bad, 2 * sizeof(long long), cudaMemcpyDeviceToHost, st));
  RD_CUDA(cudaStreamSynchronize(st));
  const long long len = off[1] - off[0];
  if (len > 0 && name_cap > 0)
    RD_CUDA(cudaMemcpyAsync(name, r->eq_names + off[0], (size_t)(len < name_cap ? len : name_cap), cudaMemcpyDeviceToHost, st));
  RD_CUDA(cudaStreamSynchronize(st));
  *name_len = len;
  return C2V_OK;
}

int c2v_reader_eval_words(const c2v_reader* r, const char** words, const int64_t** word_off, int32_t* n_words) {
  if (!r || !words || !word_off || !n_words) return rfail(C2V_ERR_INVALID, "c2v_reader_eval_words: NULL argument");
  if (!r->tab_mem) return rfail(C2V_ERR_STATE, "c2v_reader_eval_words: upload the tables first (c2v_reader_eval_tables)");
  *words = (const char*)r->tab.words;
  *word_off = (const int64_t*)r->tab.word_off;
  *n_words = r->tab.Y;
  return C2V_OK;
}

int c2v_reader_eval_score(const c2v_reader* r, const int32_t* ids, int32_t n, int32_t k, const int64_t* name_off,
                          const char* names, int32_t* rank, int32_t* first, int32_t* flags, int64_t* acc, void* stream) {
  if (!r || !ids || !name_off || !names || !rank || !first || !flags || !acc)
    return rfail(C2V_ERR_INVALID, "c2v_reader_eval_score: NULL argument");
  if (n < 1 || k < 1) return rfail(C2V_ERR_INVALID, "c2v_reader_eval_score: need n >= 1 and k >= 1");
  if (!r->tab_mem) return rfail(C2V_ERR_STATE, "c2v_reader_eval_score: upload the tables first (c2v_reader_eval_tables)");
  RD_CUDA(cudaSetDevice(r->device));
  cudaStream_t st = (cudaStream_t)stream;
  RD_CUDA(cudaMemsetAsync(acc, 0, (size_t)(k + 4) * sizeof(int64_t), st));
  eval_score_kernel<<<row_grid(r, n), 256, 0, st>>>(r->tab, ids, n, k, (const long long*)name_off,
                                                    (const unsigned char*)names, rank, first, flags,
                                                    (unsigned long long*)acc);
  RD_CUDA(cudaGetLastError());
  return C2V_OK;
}

int64_t c2v_reader_live_rows(const c2v_reader* r) { return r ? r->live : -1; }

size_t c2v_reader_device_bytes(const c2v_reader* r) { return r ? r->bytes : 0; }

}  // extern "C"
