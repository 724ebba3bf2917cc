// The lines of `<corpus>.name_scores` and `<corpus>.nearest` formatted on the device (include/c2v_b200.h "Corpus text",
// DESIGN.md §6o), byte for byte what name_scores.format_line and similarity.format_nearest_line write.  One thread per
// row writes its line twice over: a length pass, an inclusive scan of the lengths (cub), then a write pass into the
// output when the text fits.  Floats are Python's '%f' (format_fixed6, float_text.cuh, as predict.cu prints them).
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

#include <cub/device/device_scan.cuh>
#include <string>

#include "../../include/c2v_b200.h"
#include "float_text.cuh"

namespace c2v {
void set_global_error(const std::string& msg);     // engine.cu: the message c2v_last_error(NULL) returns
}

namespace {

constexpr int kThreads = 256;

int cfail(int code, const std::string& msg) {
  c2v::set_global_error(msg);
  return code;
}
#define CT_CHECK(fn, expr)                                                                                   \
  do {                                                                                                       \
    cudaError_t _c = (expr);                                                                                 \
    if (_c != cudaSuccess) return cfail(C2V_ERR_CUDA, std::string(fn) + ": " + cudaGetErrorString(_c));      \
  } while (0)

struct Out {
  char* o;
  long long len;
  __device__ void put(const char* s, long long n) {
    if (o)
      for (long long i = 0; i < n; ++i) o[len + i] = s[i];
    len += n;
  }
  __device__ void put(char c) {
    if (o) o[len] = c;
    ++len;
  }
  __device__ void put_int(long long v) {       // "%d"
    char d[20];
    int n = 0;
    const bool neg = v < 0;
    unsigned long long u = neg ? 0ull - (unsigned long long)v : (unsigned long long)v;
    do {
      d[n++] = (char)('0' + u % 10);
      u /= 10;
    } while (u);
    if (neg) put('-');
    while (n > 0) put(d[--n]);
  }
  __device__ void put_fixed(float x) {         // "%f" % float(x)
    char num[kFixedBytes];
    put(num, format_fixed6(x, num));
  }
};

// ---- name scores ---------------------------------------------------------------------------------------------------
struct ScoreArgs {
  int n;
  const char* names;
  const long long* name_off;
  const int32_t *target, *rank, *top1;
  const float *logp, *top1_logp;
  int oov;
  const char* words;
  const long long* word_off;
  int n_words;
  long long* row_end;
  char* out;
  long long cap;
};

// name \t rank \t logp \t top1_name \t top1_logp \n; '-' for the rank and logp of a name outside the vocabulary (its
// target is the OOV word) and for rank 0 (a row whose logits hold a NaN); a top1 outside the table prints the OOV word
__device__ long long score_line(const ScoreArgs& a, int r, char* o) {
  Out e{o, 0};
  e.put(a.names + a.name_off[r], a.name_off[r + 1] - a.name_off[r]);
  e.put('\t');
  const bool in_vocab = a.target[r] != a.oov;
  if (in_vocab && a.rank[r] > 0) e.put_int(a.rank[r]); else e.put('-');
  e.put('\t');
  if (in_vocab) e.put_fixed(a.logp[r]); else e.put('-');
  e.put('\t');
  const int t = (a.top1[r] >= 0 && a.top1[r] < a.n_words) ? a.top1[r] : a.oov;
  e.put(a.words + a.word_off[t], a.word_off[t + 1] - a.word_off[t]);
  e.put('\t');
  e.put_fixed(a.top1_logp[r]);
  e.put('\n');
  return e.len;
}

__global__ void __launch_bounds__(kThreads) score_len_kernel(const __grid_constant__ ScoreArgs a) {
  const int r = blockIdx.x * kThreads + threadIdx.x;
  if (r < a.n) a.row_end[r] = score_line(a, r, nullptr);
}

__global__ void __launch_bounds__(kThreads) score_write_kernel(const __grid_constant__ ScoreArgs a) {
  const int r = blockIdx.x * kThreads + threadIdx.x;
  if (r >= a.n || a.row_end[a.n - 1] > a.cap) return;
  score_line(a, r, a.out + (r ? a.row_end[r - 1] : 0));
}

// ---- nearest -------------------------------------------------------------------------------------------------------
struct NearestArgs {
  long long first, n, rows;     // lines [first, first + n) of a corpus of `rows` rows
  int k;
  const char* names;
  const long long* name_off;    // [rows + 1]
  const int32_t* idx;           // [rows, k]
  const float* val;
  long long* row_end;
  char* out;
  long long cap;
};

// name, then \t<row>,<name of row>,<similarity> per neighbour; the INT_MAX padding (and any id outside the corpus) is skipped
__device__ long long nearest_line(const NearestArgs& a, long long r, char* o) {
  Out e{o, 0};
  e.put(a.names + a.name_off[r], a.name_off[r + 1] - a.name_off[r]);
  for (int j = 0; j < a.k; ++j) {
    const int32_t id = a.idx[r * a.k + j];
    if (id < 0 || id >= a.rows) continue;
    e.put('\t');
    e.put_int(id);
    e.put(',');
    e.put(a.names + a.name_off[id], a.name_off[id + 1] - a.name_off[id]);
    e.put(',');
    e.put_fixed(a.val[r * a.k + j]);
  }
  e.put('\n');
  return e.len;
}

__global__ void __launch_bounds__(kThreads) nearest_len_kernel(const __grid_constant__ NearestArgs a) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i < a.n) a.row_end[i] = nearest_line(a, a.first + i, nullptr);
}

__global__ void __launch_bounds__(kThreads) nearest_write_kernel(const __grid_constant__ NearestArgs a) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= a.n || a.row_end[a.n - 1] > a.cap) return;
  nearest_line(a, a.first + i, a.out + (i ? a.row_end[i - 1] : 0));
}

unsigned grid_of(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

size_t scan_bytes(long long rows) {
  size_t tb = 0;
  cub::DeviceScan::InclusiveSum(nullptr, tb, (long long*)nullptr, (long long*)nullptr, rows, (cudaStream_t)0);
  return tb;
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// the line lengths row_end = scratch[0, rows) scanned in place into line ends
int scan_lengths(const char* fn, long long rows, void* scratch, size_t scratch_bytes, cudaStream_t s) {
  long long* row_end = (long long*)scratch;
  void* tmp = (char*)scratch + align256((size_t)rows * 8);
  size_t tb = scratch_bytes - align256((size_t)rows * 8);
  CT_CHECK(fn, cub::DeviceScan::InclusiveSum(tmp, tb, row_end, row_end, rows, s));
  return C2V_OK;
}

}  // namespace

size_t c2v_corpus_text_scratch_bytes(int64_t rows) {
  if (rows < 1) return 0;
  return align256((size_t)rows * 8) + scan_bytes(rows);
}

int c2v_name_scores_text(int32_t n, const char* names, const int64_t* name_off, const int32_t* target, int32_t oov,
                         const int32_t* rank, const float* logp, const int32_t* top1, const float* top1_logp,
                         const char* words, const int64_t* word_off, int32_t n_words, void* scratch, size_t scratch_bytes,
                         char* out, int64_t out_cap, int64_t* total, void* stream) {
  static const char* fn = "c2v_name_scores_text";
  if (!names || !name_off || !target || !rank || !logp || !top1 || !top1_logp || !words || !word_off || !scratch ||
      !total || (out_cap > 0 && !out) || n < 1 || out_cap < 0)
    return cfail(C2V_ERR_INVALID, "c2v_name_scores_text: NULL argument, n < 1 or negative capacity");
  if (oov < 0 || oov >= n_words) return cfail(C2V_ERR_INVALID, "c2v_name_scores_text: oov must be a word of the table");
  if (scratch_bytes < c2v_corpus_text_scratch_bytes(n))
    return cfail(C2V_ERR_INVALID, "c2v_name_scores_text: scratch_bytes below c2v_corpus_text_scratch_bytes(n)");
  cudaStream_t s = (cudaStream_t)stream;
  long long* row_end = (long long*)scratch;
  const ScoreArgs a{n, names, (const long long*)name_off, target, rank, top1, logp, top1_logp, oov, words,
                    (const long long*)word_off, n_words, row_end, out, out_cap};
  score_len_kernel<<<grid_of(n), kThreads, 0, s>>>(a);
  CT_CHECK(fn, cudaGetLastError());
  int rc;
  if ((rc = scan_lengths(fn, n, scratch, scratch_bytes, s))) return rc;
  score_write_kernel<<<grid_of(n), kThreads, 0, s>>>(a);
  CT_CHECK(fn, cudaGetLastError());
  CT_CHECK(fn, cudaMemcpyAsync(total, row_end + n - 1, 8, cudaMemcpyDeviceToHost, s));
  return C2V_OK;
}

int c2v_nearest_text(int64_t first, int64_t n, int64_t rows, int32_t k, const char* names, const int64_t* name_off,
                     const int32_t* idx, const float* val, void* scratch, size_t scratch_bytes, char* out, int64_t out_cap,
                     int64_t* total, void* stream) {
  static const char* fn = "c2v_nearest_text";
  if (!names || !name_off || !idx || !val || !scratch || !total || (out_cap > 0 && !out) || out_cap < 0 || k < 1 ||
      n < 1 || first < 0 || first + n > rows || rows > INT_MAX)
    return cfail(C2V_ERR_INVALID, "c2v_nearest_text: NULL argument, bad sizes or rows outside [0, rows)");
  if (scratch_bytes < c2v_corpus_text_scratch_bytes(n))
    return cfail(C2V_ERR_INVALID, "c2v_nearest_text: scratch_bytes below c2v_corpus_text_scratch_bytes(n)");
  cudaStream_t s = (cudaStream_t)stream;
  long long* row_end = (long long*)scratch;
  const NearestArgs a{first, n, rows, k, names, (const long long*)name_off, idx, val, row_end, out, out_cap};
  nearest_len_kernel<<<grid_of(n), kThreads, 0, s>>>(a);
  CT_CHECK(fn, cudaGetLastError());
  int rc;
  if ((rc = scan_lengths(fn, n, scratch, scratch_bytes, s))) return rc;
  nearest_write_kernel<<<grid_of(n), kThreads, 0, s>>>(a);
  CT_CHECK(fn, cudaGetLastError());
  CT_CHECK(fn, cudaMemcpyAsync(total, row_end + n - 1, 8, cudaMemcpyDeviceToHost, s));
  return C2V_OK;
}
