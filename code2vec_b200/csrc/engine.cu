// C ABI of the path-attention engine (see include/c2v_b200.h) and the orchestration of one
// forward / train / predict pass.  Host code only launches kernels: all arithmetic of the path
// (tensorflow_model.py:197-309) runs in the kernels of sgemm.cuh / kernels.cuh / umma_gemm.cuh.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <utility>
#include <vector>

#include "../../include/c2v_b200.h"
#include "common.cuh"
#include "kernels.cuh"
#include "name_rank.cuh"
#include "sgemm.cuh"
#include "umma_gemm.cuh"

using namespace c2v;

namespace {

thread_local std::string g_create_error = "";

constexpr size_t kAlign = 256;
inline size_t align_up(size_t x, size_t a = kAlign) { return (x + a - 1) / a * a; }

constexpr int kSplitDv = 18;   // split-K slices for dv = P . Y      (K = |Y|)
constexpr int kSplitDw = 48;   // split-K slices for dW = X'^T . dU  (K = B*C)

// Carve-up of the caller-provided workspace (offsets in bytes).
struct Workspace {
  size_t H, Xg, dXg, alpha, v, dv, S, loss_b, lse, loss, part, da_part, lse_part, dl;
  size_t Xg_lo, H_lo, S_lo, tgt_hi, tgt_lo, W_hi, W_lo, v_hi, v_lo;     // 3xTF32 operand splits
  size_t WT, WT_lo, vT, vT_lo, tgtT, tgtT_lo;     // K-major copies of W, v, Ytab for ctx_fwd, dY, dv (3xTF32: hi^T, lo^T)
  size_t true_logit, rscale, v_scaled, slab_flag;                  // exp_slab schedule: row factors, scaled code vectors, {range flag, fallback count}
  size_t st_src, st_pth, st_tgt, st_mask, st_target, st_topk_idx, st_topk_val, st_code, st_attn;
  size_t nx_src, nx_pth, nx_tgt;                                  // indices of the hinted NEXT batch (host entry point)
  size_t sb_src, sb_pth, sb_tgt, sb_mask, sb_target;              // second staging set (c2v_train_batch_async double buffer)
  size_t stamp_tok, stamp_path, last_tok, last_path, lr_tab;     // lazy Adam bookkeeping
  size_t stamp_tgt, last_tgt;                                    // ... of the target table (sampled softmax)
  size_t perm, bkt_count, bkt_cursor, bkt_starts;                            // locality-sorted peer gather / scatter (sharded tables)
  size_t det_keys[2], det_vals[2], det_hist, det_offs, det_starts, det_part;  // deterministic embedding-gradient sort + reduce
  size_t samp_stamp, samp_status;                                // log-uniform sampler: per-class first-draw stamps, cap counter
  size_t total;
  size_t ldS;
  size_t ldB;     // row pitch of vT: the batch rounded up to 16 bytes, as TMA requires
};

bool dims_ok(const c2v_dims* d, std::string* why) {
  auto bad = [&](const char* m) { if (why) *why = m; return false; };
  if (!d) return bad("dims is NULL");
  if (d->token_vocab < 1 || d->path_vocab < 1 || d->target_vocab < 1) return bad("vocab sizes must be >= 1");
  if (d->embed_dim < 4 || d->embed_dim % 4) return bad("embed_dim must be a positive multiple of 4");
  if (d->code_dim < 4 || d->code_dim % 4 || d->code_dim > 1024) return bad("code_dim must be a multiple of 4 in [4, 1024]");
  if (d->max_contexts < 1) return bad("max_contexts must be >= 1");
  if (d->max_batch < 1) return bad("max_batch must be >= 1");
  if (d->top_k < 1 || d->top_k > 64) return bad("top_k must be in [1, 64]");
  if ((double)d->max_batch * d->max_contexts > 2.0e9) return bad("max_batch * max_contexts overflows int32");
  return true;
}

Workspace carve(const c2v_dims& d) {
  Workspace w{};
  const size_t N = (size_t)d.max_batch * d.max_contexts, D = d.code_dim, B = d.max_batch, X = 3 * (size_t)d.embed_dim;
  w.ldS = align_up((size_t)d.target_vocab, 64);
  w.ldB = align_up(B, 4);
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes); return o; };
  w.H = take(N * D * 4);
  w.Xg = take(N * X * 4);      // gathered context matrix X' (tf32 path), kept for dW
  w.dXg = take(N * X * 4);     // dX' (tf32 path): its scatter-add overlaps the dW GEMM, which still reads X'
  w.alpha = take(N * 4);
  w.v = take(B * D * 4);
  w.dv = take(B * D * 4);
  w.S = take(B * w.ldS * 4);
  w.loss_b = take(B * 4);
  w.lse = take(B * 4);
  w.true_logit = take(B * 4);
  w.rscale = take(B * 4);
  w.v_scaled = take(B * D * 4);
  w.slab_flag = take(64);
  w.loss = take(64);
  size_t part = (size_t)kSplitDv * B * D;
  if ((size_t)kSplitDw * X * D > part) part = (size_t)kSplitDw * X * D;
  w.part = take(part * 4);
  w.da_part = take(B * D * 4);
  w.lse_part = take(B * (size_t)umma::lse_slots(d.target_vocab) * 8);   // (max, sum exp) per (row, partial slot)
  w.dl = take(B * (size_t)(kMaxSampled + 1) * 4);     // sampled softmax: dL/dlogits [B, 1+S]
  w.st_src = take(N * 4);
  w.st_pth = take(N * 4);
  w.st_tgt = take(N * 4);
  w.st_mask = take(N * 4);
  w.nx_src = take(N * 4);
  w.nx_pth = take(N * 4);
  w.nx_tgt = take(N * 4);
  w.st_target = take(B * 4);
  w.sb_src = take(N * 4);
  w.sb_pth = take(N * 4);
  w.sb_tgt = take(N * 4);
  w.sb_mask = take(N * 4);
  w.sb_target = take(B * 4);
  w.st_topk_idx = take(B * (size_t)d.top_k * 4);
  w.st_topk_val = take(B * (size_t)d.top_k * 4);
  w.st_code = take(B * D * 4);
  w.st_attn = take(N * 4);
  w.stamp_tok = take((size_t)d.token_vocab * 4);
  w.stamp_path = take((size_t)d.path_vocab * 4);
  w.last_tok = take((size_t)d.token_vocab * 4);
  w.last_path = take((size_t)d.path_vocab * 4);
  w.lr_tab = take((size_t)kLrRing * 4);
  w.perm = take(3 * N * 4);
  w.bkt_count = take((size_t)kMaxBuckets * 4);
  w.bkt_cursor = take((size_t)kMaxBuckets * 4);
  w.bkt_starts = take((size_t)(kMaxBuckets + 1) * 4);
  w.stamp_tgt = take((size_t)d.target_vocab * 4);
  w.last_tgt = take((size_t)d.target_vocab * 4);
  // 3xTF32 (C2V_MATH_3XTF32): low parts of the GEMM operands that are produced inside a step, and the
  // (hi, lo) split of the operands that must keep their fp32 originals
  w.Xg_lo = take(N * X * 4);
  w.H_lo = take(N * D * 4);
  w.S_lo = take(B * w.ldS * 4);
  w.tgt_hi = take((size_t)d.target_vocab * D * 4);
  w.tgt_lo = take((size_t)d.target_vocab * D * 4);
  w.W_hi = take(X * D * 4);
  w.W_lo = take(X * D * 4);
  w.v_hi = take(B * D * 4);
  w.v_lo = take(B * D * 4);
  // K-major (transposed) copies of the operands the engine stores MN-major: W^T [D, 3d] for ctx_fwd, v^T [D, ldB] for dY,
  // Ytab^T [D, ldS] for dv; in 3xTF32 they hold the high parts and the *_lo regions the residuals
  w.WT = take(X * D * 4);
  w.WT_lo = take(X * D * 4);
  w.vT = take(D * w.ldB * 4);
  w.vT_lo = take(D * w.ldB * 4);
  w.tgtT = take(D * w.ldS * 4);
  w.tgtT_lo = take(D * w.ldS * 4);
  // option "deterministic": ping-pong keys / values of the 3 N entries, per-tile digit histograms and their scan, and two
  // chunk-partial slots of d floats per K entries (det_slot)
  const size_t M = 3 * N, tiles = (M + kDetSortTile - 1) / kDetSortTile;
  for (int i = 0; i < 2; ++i) { w.det_keys[i] = take(M * 4); w.det_vals[i] = take(M * 4); }
  w.det_hist = take(kDetRadix * tiles * 4);
  w.det_offs = take(kDetRadix * tiles * 4);
  w.det_starts = take((kDetRadix * tiles + 1) * 4);
  w.det_part = take(2 * ((M + kDetChunk - 1) / kDetChunk) * (size_t)d.embed_dim * 4);
  // c2v_sample_log_uniform: one 64-bit (call tag, first draw index) stamp per target class, and its cap-hit counter
  w.samp_stamp = take((size_t)d.target_vocab * 8);
  w.samp_status = take(64);
  w.total = off;
  return w;
}

}  // namespace

// Phases of a pass, for per-kernel timing (option "profile"): CUDA events bracket each phase on
// the launching stream; c2v_phase_stats() resolves them.
enum Phase { PH_CTX_FWD = 0, PH_ATTN_FWD, PH_LOGITS, PH_XENT, PH_DV, PH_DY, PH_ATTN_BWD, PH_DW, PH_DX_SCATTER,
             PH_ADAM, PH_TOPK, PH_SAMPLED, PH_GATHER, PH_DX_GEMM, PH_ADAM_CATCHUP, PH_SPLIT, PH_ADAM_SWEEP, PH_PEER_SORT, PH_INBOX_APPLY,
             PH_SAMPLER, PH_NAME_RANK, PH_COUNT };
const char* const kPhaseNames[PH_COUNT] = {"ctx_fwd", "attn_fwd", "logits", "xent", "dv", "dY", "attn_bwd", "dW",
                                           "dx_scatter", "adam", "topk", "sampled_softmax", "gather", "dx_gemm",
                                           "adam_catchup", "split", "adam_sweep", "peer_sort", "inbox_apply", "sampler",
                                           "name_rank"};
struct PhaseLog {
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> free_list;
  double total_ms = 0.0;
  int64_t count = 0;
};

// Schedule of the softmax head (logits -> cross entropy -> dL/dlogits -> dv, dY) for one call: head_schedule() picks it
enum HeadSchedule {
  HEAD_SIMT,        // fp32: SIMT logits; the fused step's xent_kernel writes P = dL/dlogits in place
  HEAD_TWO_PASS,    // logits (+ log-sum-exp partials), rewritten to P by softmax_grad_kernel
  HEAD_LOADERS,     // logits (+ partials), turned into P by the dv / dY GEMMs' A loaders (tf32, option fuse_softmax_grad)
  HEAD_RECOMPUTE,   // a log-sum-exp-only logits pass, then a second one whose epilogue writes P (option recompute_logits)
  HEAD_EXP_SLAB,    // U = exp(s - true logit), normalised by per-row factors inside dv / dY (option exp_slab)
};

// How the dv / dY GEMMs read the slab: as P, as P with row i scaled by row_scale[i] (exp_slab: dv's reduction applies the
// factor, dY's code vectors come scaled by it), or as logits that the GEMMs' A loaders turn into P (loaders, sg)
struct SlabDesc {
  const float* row_scale = nullptr;
  bool loaders = false;
  umma::SoftmaxGradArgs sg{};
};

struct PendingDy {            // a dY = P^T . v deferred into context_backward (option dy_late == 1); v == nullptr: none
  const float* v = nullptr;
  int B = 0;
  SlabDesc slab;
};

struct c2v_engine {
  PhaseLog phase[PH_COUNT];
  int profile = 0;
  c2v_dims dims;
  int device;
  Workspace ws;
  char* wbase;
  size_t wbytes;
  c2v_tensors theta, grad, am, av;
  ShardedTable th_tok{}, th_path{}, gr_tok{}, gr_path{};   // how kernels reach the two embedding tables
  int table_world = 1;       // > 1: tables are row-sharded over peers (c2v_bind_table_shards)
  float grad_scale = 1.f;
  // lazy-but-exact dense Adam for the embedding tables (option "lazy_adam")
  int lazy = 0;
  int adam_rows_occ = 4;
  int sweep_period = 32;                // lazy Adam: every step brings a 1/R slice of each table up to date, so no row
                                        // is ever more than R steps behind (bounds the replay of rarely used rows and
                                        // the cost of c2v_sync_tables); 0 = off
  int64_t full_flush_t = 0;             // step count as of which every row was last known to be current
  int rest_shortcut = 1;                // option "adam_rest_shortcut": replay_row may stop dividing once theta rests
  bool tgt_lazy = false;                // the target table's rows are updated lazily too (sampled softmax steps)
  bool tgt_t_valid = false;             // ws.tgtT (3xTF32: tgtT / tgtT_lo, as the split) holds the current target table transposed
  bool lazy_grads_pending = false;  // a train step's embedding gradients are in the tables and c2v_adam_step has not followed
  int64_t adam_t_done = 0;   // Adam steps applied so far
  int32_t mark_epoch = 0;
  float hp_lr = 0.f, hp_b1 = 0.f, hp_b2 = 0.f, hp_eps = 0.f;
  bool hp_set = false;
  bool has_theta, has_grad, has_adam;
  bool emb_grads_clean;      // token/path gradient tables are known to be all-zero
  int math_mode;
  const int32_t* sorted_src = nullptr;   // ws.perm / ws.bkt_starts hold the bucket order of THIS batch (set by the forward pass)
  int sorted_rows = 0;
  InboxSet inbox{};          // push-based gradient exchange (c2v_bind_scatter_inbox); world == 0: not bound
  int ordered_exchange = 0;  // option "ordered_exchange": sharded tables take sorted per-row sums through the inbox, folded in rank order
  bool exchange_pushed = false;   // ws.det_starts holds the bounds of an ordered push (option "ordered_exchange_rows")
  int sort_peer = 1;         // option "sort_peer_access": sharded tables are gathered / scattered in (owner, 2 MB page) order
  bool bkt_zeroed = false;   // the bucket counters have been cleared once (bucket_scan_kernel leaves them cleared)
  int recompute = 0;         // option "recompute_logits" (tensor-core modes, single-GPU step): the logits GEMM runs twice -- once for the
                             // log-sum-exp only, once writing dL/dlogits from its epilogue -- instead of writing logits and rewriting them.
                             // In 3xTF32 it costs a third 3x GEMM and a second table split: off by default
  int exp_slab = 1;          // option "exp_slab" (tensor-core modes, single-GPU full-softmax step; default on): the logits epilogue writes
                             // U = exp(s - true logit) and the softmax's normalisation is deferred into per-row factors applied by the
                             // dv / dY GEMMs, so no pass re-reads the slab to turn logits into dL/dlogits (DESIGN.md section 4.9).  Rows
                             // outside the fp32 window make that step fall back, on the device, to the two-pass schedule.
  bool slab_flag_zeroed = false;
  HeadSchedule split_fwd = HEAD_SIMT;   // schedule of the last c2v_target_forward, for c2v_target_backward (HEAD_SIMT once consumed)
  int gather_occ[2] = {0, 0};         // resident CTAs per SM of gather_ctx_kernel<false / true>, queried once
  int adam_epi_prefetch = 0; // option "adam_epilogue_prefetch" (off by default): the dY epilogue's Adam update prefetches its (theta, m, v)
                             // lines into L2 one tile ahead
  int fuse_sg = 0;           // option "fuse_softmax_grad": dv / dY compute dL/dlogits from the logits slab on the fly (tf32 mode):
                             // the GEMM's loaders transform each A element on its way into shared memory, which removes the 2.1 GB
                             // softmax-gradient pass but takes the A operand off TMA; off by default
  int fuse_gather = 0;       // option "fuse_gather": gather -> projection -> tanh as one kernel on the tf32 path (umma::launch_ctx_fused);
                             // bit-identical to the two-kernel path; off by default
  int cta_pair = 2;          // option "cta_pair": accepted and validated, no effect (the sm_90a GEMM has no CTA-pair form)
  int num_sms;
  cudaEvent_t ev_tgt_ready = nullptr;   // recorded after dY (caller-owned)
  int dy_late = 1;                      // where dY = P^T.v runs: 0 after dv, 1 inside context_backward, 2 on side2 after dv
  PendingDy pending_dy;
  cudaStream_t side = nullptr;          // engine-owned: the embedding scatter-add runs here, next to the dY / dW GEMMs
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  cudaStream_t copy = nullptr;          // engine-owned: host -> device copies of c2v_train_batch_async
  cudaEvent_t ev_h2d[2] = {nullptr, nullptr}, ev_used[2] = {nullptr, nullptr};
  bool used_valid[2] = {false, false};
  uint64_t async_n = 0;
  cudaStream_t side2 = nullptr;         // engine-owned: the dY (+ target Adam) GEMM with dy_late == 2
  cudaEvent_t ev_fork2 = nullptr, ev_join2 = nullptr;
  bool dy_in_flight = false;            // a dY launched on side2 has not been joined yet
  // target-table Adam folded into the dY epilogue (c2v_arm_target_adam)
  bool tgt_armed = false;               // the next tensor-core dY product applies the update instead of storing dY
  float tgt_lr = 0.f, tgt_b1 = 0.f, tgt_b2 = 0.f, tgt_eps = 0.f;
  int64_t tgt_t = 0;
  int64_t armed_t = 0;                  // step whose hyper-parameters c2v_arm_target_adam declared (0 = none)
  // next-batch hint (c2v_hint_next_batch): the deferred embedding-row updates of the NEXT batch's rows are
  // applied on the side stream during this step's backward, next to the dY / dW GEMMs
  const int32_t* hint_src = nullptr;
  const int32_t* hint_pth = nullptr;
  const int32_t* hint_tgt = nullptr;
  int hint_B = 0;
  int64_t early_t = 0;                  // step count the early catch-up already assumed applied (0 = none)
  int64_t early_count = 0;              // how many steps used the hint (option "early_catchup_count", read-only)
  int fuse_tgt = 0;                     // option "fuse_target_adam": c2v_train_batch_host arms itself
  int64_t tgt_fused_t = 0;              // step count whose target update has already been applied (0 = none)
  uint32_t sample_tag = 0;              // c2v_sample_log_uniform: tag of the last call (counts down; 0 = stamps not initialised)
  bool cap_hits_zeroed = false;         // the sampler's cap-hit counter (workspace) has been cleared
  unsigned long long* vstamp = nullptr; // c2v_sample_log_uniform_vocab: first-draw stamps of vstamp_Y classes (own allocation)
  int32_t vstamp_Y = 0;
  uint32_t vsample_tag = 0;             // as sample_tag, for vstamp
  int deterministic;
  int64_t launches;
  std::string err;
};

namespace {

int fail(c2v_engine* e, int code, const std::string& msg) {
  if (e) e->err = msg; else g_create_error = msg;
  return code;
}

struct PhaseTimer {
  c2v_engine* e; int ph; cudaStream_t st; cudaEvent_t stop = nullptr;
  PhaseTimer(c2v_engine* e_, int ph_, cudaStream_t st_) : e(e_), ph(ph_), st(st_) {
    if (!e->profile) return;
    PhaseLog& L = e->phase[ph];
    std::pair<cudaEvent_t, cudaEvent_t> ev;
    if (!L.free_list.empty()) { ev = L.free_list.back(); L.free_list.pop_back(); }
    else { cudaEventCreate(&ev.first); cudaEventCreate(&ev.second); }
    cudaEventRecord(ev.first, st);
    stop = ev.second;
    L.pending.push_back(ev);
  }
  ~PhaseTimer() { if (stop) cudaEventRecord(stop, st); }
};

#define C2V_CUDA(e, expr)                                                                         \
  do {                                                                                            \
    cudaError_t _c = (expr);                                                                      \
    if (_c != cudaSuccess)                                                                        \
      return fail((e), C2V_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_c));         \
  } while (0)

// every kernel launch goes through this so the launch counter is truthful
#define C2V_LAUNCH(e, ...)                                                                        \
  do {                                                                                            \
    __VA_ARGS__;                                                                                  \
    cudaError_t _c = cudaGetLastError();                                                          \
    if (_c != cudaSuccess)                                                                        \
      return fail((e), C2V_ERR_CUDA, std::string("kernel launch failed: ") + cudaGetErrorString(_c)); \
    (e)->launches++;                                                                              \
  } while (0)

// adam_rows_kernel as one wave of num_sms * occupancy blocks (option "adam_rows_occupancy": 4 or 5)
#define C2V_ADAM_ROWS(e, MODE, stream, ...)                                                                    \
  do {                                                                                                         \
    if ((e)->adam_rows_occ == 5)                                                                               \
      C2V_LAUNCH(e, (adam_rows_kernel<MODE, 5><<<(e)->num_sms * 5, 256, 0, stream>>>(__VA_ARGS__)));           \
    else                                                                                                       \
      C2V_LAUNCH(e, (adam_rows_kernel<MODE, 4><<<(e)->num_sms * 4, 256, 0, stream>>>(__VA_ARGS__)));           \
  } while (0)

// the "theta rests" exit of the row replay (kernels.cuh, replay_row) is proven for these hyper-parameter ranges only
inline int rest_ok(const c2v_engine* e) {
  return (e->rest_shortcut && e->hp_b1 > 0.f && e->hp_b1 <= 0.95f && e->hp_b2 >= 0.99f && e->hp_b2 < 1.f && e->hp_eps > 0.f) ? 1 : 0;
}
// adam_move's zero-numerator exit (common.cuh) matches the division only while sqrt(v) + eps > 0, i.e. for eps > 0
inline int pos_eps(const c2v_engine* e) { return e->hp_eps > 0.f ? 1 : 0; }
inline bool is_tc(const c2v_engine* e) { return e->math_mode != C2V_MATH_FP32; }          // tensor-core (wgmma) GEMMs
inline bool is_3x(const c2v_engine* e) { return e->math_mode == C2V_MATH_3XTF32; }        // ... as 3xTF32
inline bool aligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }

enum HeadApi { API_STEP, API_TARGET_FORWARD, API_TARGET_BACKWARD, API_LOSS };

// The one place that decides the softmax head's schedule, for the API asking and its code vectors v:
//   fused step       fp32 -> SIMT; recompute_logits -> RECOMPUTE (wins over exp_slab); exp_slab -> EXP_SLAB (both only
//                    without fuse_softmax_grad); tf32 with fuse_softmax_grad -> LOADERS; otherwise TWO_PASS
//   target_forward   tensor core, v 16-B aligned, exp_slab, not fuse_softmax_grad, grads bound -> EXP_SLAB (recompute_logits
//                    does not apply here); otherwise TWO_PASS (lse partials) if tensor core and aligned, else SIMT
//   target_backward  the forward left U in the slab -> EXP_SLAB; otherwise tf32 with fuse_softmax_grad -> LOADERS, else
//                    softmax_grad_kernel<3xTF32> rewrites the slab (TWO_PASS, SIMT in fp32)
//   c2v_loss         tensor core and aligned -> TWO_PASS (lse partials + xent_combine_kernel), else SIMT (xent_kernel)
// run_logits sends a call that is not on the tensor cores to the SIMT GEMM, which only stores logits: none of the
// schedules above asks it for more.
HeadSchedule head_schedule(const c2v_engine* e, HeadApi api, const float* v) {
  const bool tc_aligned = is_tc(e) && aligned16(v);
  switch (api) {
    case API_STEP:
      if (!is_tc(e)) return HEAD_SIMT;
      if (e->recompute && !e->fuse_sg) return HEAD_RECOMPUTE;
      if (e->exp_slab && !e->fuse_sg) return HEAD_EXP_SLAB;
      return (e->fuse_sg && !is_3x(e)) ? HEAD_LOADERS : HEAD_TWO_PASS;
    case API_TARGET_FORWARD:
      if (!tc_aligned) return HEAD_SIMT;
      return (e->exp_slab && !e->fuse_sg && e->has_grad) ? HEAD_EXP_SLAB : HEAD_TWO_PASS;
    case API_TARGET_BACKWARD:
      if (e->split_fwd == HEAD_EXP_SLAB) return HEAD_EXP_SLAB;
      if (!is_tc(e)) return HEAD_SIMT;
      return (e->fuse_sg && !is_3x(e)) ? HEAD_LOADERS : HEAD_TWO_PASS;
    case API_LOSS:
      return tc_aligned ? HEAD_TWO_PASS : HEAD_SIMT;
  }
  return HEAD_SIMT;
}

template <class T> T* wsp(c2v_engine* e, size_t off) { return reinterpret_cast<T*>(e->wbase + off); }

inline bool has_all(const c2v_tensors* t) { return t && t->tok && t->path && t->tgt && t->W && t->a; }

Dropout make_dropout(const c2v_dims& d, float keep, uint64_t seed, uint64_t step, const float* ext) {
  Dropout dp{};
  dp.ctx_dim = 3 * d.embed_dim;
  dp.enabled = (keep < 1.0f) ? 1 : 0;
  dp.ext = ext;
  dp.scale = 1.0f / keep;
  double thr = (double)keep * 4294967296.0;
  dp.thr = thr >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)thr;
  dp.key = make_uint2((uint32_t)(seed & 0xFFFFFFFFull), (uint32_t)(seed >> 32));
  dp.step = make_uint2((uint32_t)(step & 0xFFFFFFFFull), (uint32_t)(step >> 32));
  return dp;
}

int check_batch(c2v_engine* e, int32_t B) {
  if (!e) return C2V_ERR_INVALID;
  if (B < 1 || B > e->dims.max_batch) return fail(e, C2V_ERR_INVALID, "batch size out of range [1, max_batch]");
  if (!e->wbase) return fail(e, C2V_ERR_STATE, "workspace not bound (c2v_bind_workspace)");
  if (!e->has_theta) return fail(e, C2V_ERR_STATE, "parameters not bound (c2v_bind_params)");
  return C2V_OK;
}

// ---- attention kernels: dispatch on ceil(D / 128) ------------------------------------------------
int launch_attn_fwd(c2v_engine* e, cudaStream_t st, const float* H, const float* mask, int B, float* alpha, float* v) {
  const int C = e->dims.max_contexts, D = e->dims.code_dim;
  const size_t smem = ((size_t)((C + 3) & ~3) + 32 + kAttnWarps + (size_t)kAttnWarps * D) * sizeof(float);
  const float* a = e->theta.a;
  PhaseTimer pt(e, PH_ATTN_FWD, st);
#define C2V_AF(NV)                                                                                        \
  do {                                                                                                    \
    if (smem > 48 * 1024)                                                                                 \
      C2V_CUDA(e, cudaFuncSetAttribute(attn_fwd_kernel<NV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    C2V_LAUNCH(e, (attn_fwd_kernel<NV><<<B, kAttnThreads, smem, st>>>(H, a, mask, C, D, alpha, v)));      \
  } while (0)
  switch ((D + 127) / 128) {
    case 1: C2V_AF(1); break;
    case 2: C2V_AF(2); break;
    case 3: C2V_AF(3); break;
    case 4: C2V_AF(4); break;
    case 5: case 6: C2V_AF(6); break;
    default: C2V_AF(8); break;
  }
#undef C2V_AF
  return C2V_OK;
}

// v: the code vectors the forward pass produced for these examples (ws.v)
int launch_attn_bwd(c2v_engine* e, cudaStream_t st, float* H, const float* alpha, const float* dv, const float* v, int B,
                    float* da_part, float* H_lo) {
  const int C = e->dims.max_contexts, D = e->dims.code_dim;
  const size_t smem = (size_t)kAttnWarps * D * sizeof(float);
  const float* a = e->theta.a;
  PhaseTimer pt(e, PH_ATTN_BWD, st);
#define C2V_AB(NV)                                                                                        \
  do {                                                                                                    \
    if (H_lo) {                                                                                           \
      if (smem > 48 * 1024)                                                                               \
        C2V_CUDA(e, cudaFuncSetAttribute(attn_bwd_kernel<NV, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
      C2V_LAUNCH(e, (attn_bwd_kernel<NV, true><<<B, kAttnThreads, smem, st>>>(H, alpha, dv, v, a, C, D, da_part, H_lo))); \
    } else {                                                                                              \
      if (smem > 48 * 1024)                                                                               \
        C2V_CUDA(e, cudaFuncSetAttribute(attn_bwd_kernel<NV, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
      C2V_LAUNCH(e, (attn_bwd_kernel<NV, false><<<B, kAttnThreads, smem, st>>>(H, alpha, dv, v, a, C, D, da_part, nullptr))); \
    }                                                                                                     \
  } while (0)
  switch ((D + 127) / 128) {
    case 1: C2V_AB(1); break;
    case 2: C2V_AB(2); break;
    case 3: C2V_AB(3); break;
    case 4: C2V_AB(4); break;
    case 5: case 6: C2V_AB(6); break;
    default: C2V_AB(8); break;
  }
#undef C2V_AB
  return C2V_OK;
}

// row_scale (optional): the n results are rows of length row_len; row i is multiplied by row_scale[i]
int launch_colsum(c2v_engine* e, cudaStream_t st, const float* in, size_t stride, int R, int n, float* out,
                  const float* row_scale = nullptr, int row_len = 0) {
  if (R <= 64 && n % 4 == 0 && stride % 4 == 0 && (!row_scale || row_len % 4 == 0)) {          // split-K slices: few rows, many columns
    size_t blocks = ((size_t)n / 4 + 255) / 256;
    if (blocks > (size_t)e->num_sms * 16) blocks = (size_t)e->num_sms * 16;
    C2V_LAUNCH(e, (slice_sum_kernel<<<(unsigned)blocks, 256, 0, st>>>(in, stride, R, (size_t)n / 4, out, row_scale, row_scale ? row_len / 4 : 1)));
    return C2V_OK;
  }
  C2V_LAUNCH(e, (colsum_kernel<<<(n + 31) / 32, dim3(32, 32), 0, st>>>(in, stride, R, n, out)));
  if (row_scale) C2V_LAUNCH(e, (scale_rows_kernel<<<(unsigned)(((size_t)n + 255) / 256), 256, 0, st>>>(out, row_scale, out, row_len, (size_t)n)));
  return C2V_OK;
}

ContextSource make_source(c2v_engine* e, const int32_t* src, const int32_t* pth, const int32_t* tgt, int B) {
  ContextSource cs{};
  cs.src = src; cs.pth = pth; cs.tgt = tgt;
  cs.tok = e->th_tok; cs.path = e->th_path;
  cs.d = e->dims.embed_dim;
  cs.rows = B * e->dims.max_contexts;
  return cs;
}

// Lazy Adam: stamp the rows this batch references and replay their pending zero-gradient steps so the
// gather below reads exactly what a dense Adam would have left there.
int prepare_rows(c2v_engine* e, cudaStream_t st, const ContextSource& cs) {
  if (!e->lazy) return C2V_OK;
  PhaseTimer pt(e, PH_ADAM_CATCHUP, st);
  const c2v_dims& d = e->dims;
  int32_t* stamp_tok = wsp<int32_t>(e, e->ws.stamp_tok);
  int32_t* stamp_path = wsp<int32_t>(e, e->ws.stamp_path);
  e->mark_epoch++;
  C2V_LAUNCH(e, (mark_rows_kernel<<<(cs.rows + 255) / 256, 256, 0, st>>>(cs.src, cs.pth, cs.tgt, cs.rows, stamp_tok, stamp_path,
                                                                        e->mark_epoch)));
  if (e->adam_t_done > 0) {
    const float* lr_tab = wsp<float>(e, e->ws.lr_tab);
    C2V_ADAM_ROWS(e, ADAM_ROWS_CATCHUP, st,
                  e->theta.tok, e->grad.tok, e->am.tok, e->av.tok, d.token_vocab, d.embed_dim, stamp_tok, e->mark_epoch,
                      wsp<int32_t>(e, e->ws.last_tok), (int32_t)e->adam_t_done, lr_tab, e->hp_b1, e->hp_b2, e->hp_eps, rest_ok(e), pos_eps(e));
    C2V_ADAM_ROWS(e, ADAM_ROWS_CATCHUP, st,
                  e->theta.path, e->grad.path, e->am.path, e->av.path, d.path_vocab, d.embed_dim, stamp_path, e->mark_epoch,
                      wsp<int32_t>(e, e->ws.last_path), (int32_t)e->adam_t_done, lr_tab, e->hp_b1, e->hp_b2, e->hp_eps, rest_ok(e), pos_eps(e));
  }
  return C2V_OK;
}

// every row of one table that is behind step t: replay (one warp per row)
int launch_sweep(c2v_engine* e, cudaStream_t st, float* p, float* g, float* m, float* v, int rows, int dim, int32_t* last, int64_t t) {
  if (rows <= 0) return C2V_OK;
  int blocks = (rows + 7) / 8;
  if (blocks > e->num_sms * 4) blocks = e->num_sms * 4;
  C2V_LAUNCH(e, (adam_sweep_kernel<4><<<blocks, 256, 0, st>>>(p, g, m, v, rows, dim, last, (int32_t)t, wsp<float>(e, e->ws.lr_tab), e->hp_b1,
                                                             e->hp_b2, e->hp_eps, rest_ok(e), pos_eps(e))));
  return C2V_OK;
}

// Lazy Adam: bring every row of both embedding tables up to date (export, checkpoint, mode switches).
int flush_rows(c2v_engine* e, cudaStream_t st) {
  if (!e->lazy || e->adam_t_done == 0) return C2V_OK;
  const c2v_dims& d = e->dims;
  const float* lr_tab = wsp<float>(e, e->ws.lr_tab);
  { int rcw = launch_sweep(e, st, e->theta.tok, e->grad.tok, e->am.tok, e->av.tok, d.token_vocab, d.embed_dim, wsp<int32_t>(e, e->ws.last_tok), e->adam_t_done);
    if (rcw) return rcw; }
  { int rcw = launch_sweep(e, st, e->theta.path, e->grad.path, e->am.path, e->av.path, d.path_vocab, d.embed_dim, wsp<int32_t>(e, e->ws.last_path), e->adam_t_done);
    if (rcw) return rcw; }
  if (e->tgt_lazy)
    { int rcw = launch_sweep(e, st, e->theta.tgt, e->grad.tgt, e->am.tgt, e->av.tgt, d.target_vocab, d.code_dim, wsp<int32_t>(e, e->ws.last_tgt), e->adam_t_done);
    if (rcw) return rcw; }
  e->full_flush_t = e->adam_t_done;
  return C2V_OK;
}

// The target table leaves the lazily updated set (a full-softmax step, a full-vocabulary read): bring its rows
// up to date first.  Its gradient rows are zero afterwards (cleared as they are applied).
int end_target_lazy(c2v_engine* e, cudaStream_t st) {
  if (!e->tgt_lazy) return C2V_OK;
  if (e->adam_t_done > 0) {
    const c2v_dims& d = e->dims;
    { int rcw = launch_sweep(e, st, e->theta.tgt, e->grad.tgt, e->am.tgt, e->av.tgt, d.target_vocab, d.code_dim, wsp<int32_t>(e, e->ws.last_tgt), e->adam_t_done);
    if (rcw) return rcw; }
  }
  e->tgt_lazy = false;
  return C2V_OK;
}

// Lazy Adam sweep: rows [rows*ph/R, rows*(ph+1)/R) of every lazily updated table are brought up to date each
// step (ph = t mod R), so a row is never more than R steps behind whatever the data looks like: the replay
// of a rarely referenced row costs at most R iterations, and c2v_sync_tables at most R per row.
int sweep_rows(c2v_engine* e, cudaStream_t st, int64_t t) {
  const int R = e->sweep_period;
  if (!e->lazy || R <= 0) return C2V_OK;
  if (R == 1) return flush_rows(e, st);
  PhaseTimer pt(e, PH_ADAM_SWEEP, st);
  const c2v_dims& d = e->dims;
  const float* lr_tab = wsp<float>(e, e->ws.lr_tab);
  const int64_t ph = t % R;
  auto slice = [&](float* p, float* g, float* m, float* v, int rows, int dim, int32_t* last) -> int {
    const int64_t lo = (int64_t)rows * ph / R, hi = (int64_t)rows * (ph + 1) / R;
    if (hi <= lo) return C2V_OK;
    const size_t o = (size_t)lo * dim;
    return launch_sweep(e, st, p + o, g + o, m + o, v + o, (int)(hi - lo), dim, last + lo, t);
  };
  int rc;
  if ((rc = slice(e->theta.tok, e->grad.tok, e->am.tok, e->av.tok, d.token_vocab, d.embed_dim, wsp<int32_t>(e, e->ws.last_tok)))) return rc;
  if ((rc = slice(e->theta.path, e->grad.path, e->am.path, e->av.path, d.path_vocab, d.embed_dim, wsp<int32_t>(e, e->ws.last_path)))) return rc;
  if (e->tgt_lazy &&
      (rc = slice(e->theta.tgt, e->grad.tgt, e->am.tgt, e->av.tgt, d.target_vocab, d.code_dim, wsp<int32_t>(e, e->ws.last_tgt)))) return rc;
  if (ph == R - 1) e->full_flush_t = t - R + 1;      // every row has been visited at or after step t - R + 1
  return C2V_OK;
}

// Lazy Adam + next-batch hint: once this step's scatter-add is queued on the side stream, the rows the NEXT
// batch references can already be brought up to date through THIS step (its hyper-parameters are known
// from c2v_arm_target_adam): their deferred updates then run next to the dY / dW GEMMs instead of at the
// head of the next step.  Same kernels, same arithmetic, only earlier; anything not covered here is
// handled by the next step's prepare_rows as usual.
int early_catchup(c2v_engine* e, cudaStream_t side) {
  const int32_t *hs = e->hint_src, *hp = e->hint_pth, *ht = e->hint_tgt;
  const int hB = e->hint_B;
  e->hint_src = e->hint_pth = e->hint_tgt = nullptr;          // one-shot
  e->hint_B = 0;
  if (!hs || !e->lazy || e->table_world > 1) return C2V_OK;
  const int64_t t = e->armed_t;
  if (t != e->adam_t_done + 1) return C2V_OK;
  // pending steps were recorded under e->hp_*: only valid to run ahead if this step keeps them
  if (!e->hp_set || e->tgt_lr != e->hp_lr || e->tgt_b1 != e->hp_b1 || e->tgt_b2 != e->hp_b2 || e->tgt_eps != e->hp_eps)
    return C2V_OK;
  const c2v_dims& d = e->dims;
  const double lr_t = (double)e->tgt_lr * sqrt(1.0 - pow((double)e->tgt_b2, (double)t)) / (1.0 - pow((double)e->tgt_b1, (double)t));
  float* lr_tab = wsp<float>(e, e->ws.lr_tab);
  int32_t* stamp_tok = wsp<int32_t>(e, e->ws.stamp_tok);
  int32_t* stamp_path = wsp<int32_t>(e, e->ws.stamp_path);
  PhaseTimer pt(e, PH_ADAM_CATCHUP, side);
  C2V_LAUNCH(e, (set_float_kernel<<<1, 1, 0, side>>>(lr_tab + (t & kLrRingMask), (float)lr_t)));
  e->mark_epoch++;
  const int rows = hB * d.max_contexts;
  C2V_LAUNCH(e, (mark_rows_kernel<<<(rows + 255) / 256, 256, 0, side>>>(hs, hp, ht, rows, stamp_tok, stamp_path, e->mark_epoch)));
  C2V_ADAM_ROWS(e, ADAM_ROWS_CATCHUP, side,
                  e->theta.tok, e->grad.tok, e->am.tok, e->av.tok, d.token_vocab, d.embed_dim, stamp_tok, e->mark_epoch,
                    wsp<int32_t>(e, e->ws.last_tok), (int32_t)t, lr_tab, e->hp_b1, e->hp_b2, e->hp_eps, rest_ok(e), pos_eps(e));
  C2V_ADAM_ROWS(e, ADAM_ROWS_CATCHUP, side,
                  e->theta.path, e->grad.path, e->am.path, e->av.path, d.path_vocab, d.embed_dim, stamp_path, e->mark_epoch,
                    wsp<int32_t>(e, e->ws.last_path), (int32_t)t, lr_tab, e->hp_b1, e->hp_b2, e->hp_eps, rest_ok(e), pos_eps(e));
  e->early_t = t;
  e->early_count++;
  return C2V_OK;
}

// 3xTF32: (hi, lo) tf32 split of a whole fp32 buffer into two workspace regions.
int split_small(c2v_engine* e, cudaStream_t st, const float* x, size_t n, size_t off_hi, size_t off_lo) {
  PhaseTimer pt(e, PH_SPLIT, st);
  const size_t n4 = n / 4;                 // every split buffer here is a multiple of 4 floats (dims_ok)
  size_t blocks = (n4 + 255) / 256;
  if (blocks > (size_t)e->num_sms * 16) blocks = (size_t)e->num_sms * 16;
  if (blocks < 1) blocks = 1;
  C2V_LAUNCH(e, (split_tf32_kernel<<<(unsigned)blocks, 256, 0, st>>>(x, wsp<float>(e, off_hi), wsp<float>(e, off_lo), n4)));
  return C2V_OK;
}

// K-major copy [cols, ldT] (workspace region off_t) of a row-major operand x [rows, cols] that a GEMM reads MN-major.  split
// (3xTF32): the transposed tf32 split goes to off_t / off_lo, and the untransposed one to hi / lo when they are given.
int transpose_operand(c2v_engine* e, cudaStream_t st, const float* x, int rows, int cols, size_t ldT, size_t off_t, bool split,
                      size_t off_lo = 0, float* hi = nullptr, float* lo = nullptr) {
  const dim3 grid((unsigned)((rows + 31) / 32), (unsigned)((cols + 31) / 32));
  if (split)
    C2V_LAUNCH(e, (transpose_kernel<true><<<grid, 256, 0, st>>>(x, rows, cols, wsp<float>(e, off_t), wsp<float>(e, off_lo), ldT, hi, lo)));
  else
    C2V_LAUNCH(e, (transpose_kernel<false><<<grid, 256, 0, st>>>(x, rows, cols, wsp<float>(e, off_t), nullptr, ldT, nullptr, nullptr)));
  return C2V_OK;
}

// Ytab^T for dv, from the current target table (every row must be current: callers run end_target_lazy first); 3xTF32: as
// its transposed split.  A training step's logits GEMM writes it from its B tiles (launch_logits, for_dv); this pass is for
// a dv that no such logits pass preceded.
int transpose_table(c2v_engine* e, cudaStream_t st) {
  const int Y = e->dims.target_vocab, D = e->dims.code_dim;
  int rc;
  if (is_3x(e)) {
    PhaseTimer pt(e, PH_SPLIT, st);
    rc = transpose_operand(e, st, e->theta.tgt, Y, D, e->ws.ldS, e->ws.tgtT, true, e->ws.tgtT_lo);
  } else {
    PhaseTimer pt(e, PH_DV, st);
    rc = transpose_operand(e, st, e->theta.tgt, Y, D, e->ws.ldS, e->ws.tgtT, false);
  }
  if (rc) return rc;
  e->tgt_t_valid = true;
  return C2V_OK;
}

// Sharded tables: bucket the batch's 3 B C context entries by (owner rank, 2 MB page of the owner's shard) into ws.perm.
// Returns false when the plan does not apply (tables not sharded, option off, too many buckets).
bool plan_buckets(c2v_engine* e, BucketPlan* bp, bool force = false) {
  if (e->table_world <= 1) return false;
  const c2v_dims& d = e->dims;
  // sort_peer_access: 0 never, 1 (default) when the tables are large enough for random peer accesses to thrash the TLB
  // (the 2 GB threshold below), 2 always; the inbox exchange always needs the order
  const double table_bytes = ((double)d.token_vocab + d.path_vocab) * d.embed_dim * 4.0;
  if (!force && (e->sort_peer == 0 || (e->sort_peer == 1 && table_bytes < 2.0e9))) return false;
  const int W = e->table_world;
  int rows_per_page = (int)((2u << 20) / ((size_t)d.embed_dim * 4));
  int ps = 0;
  while ((2 << ps) <= rows_per_page) ++ps;
  bp->shift = e->th_tok.shift; bp->mask = e->th_tok.mask; bp->page_shift = ps;
  const int rows_tok = (d.token_vocab + W - 1) / W, rows_path = (d.path_vocab + W - 1) / W;
  bp->pages_tok = (rows_tok >> ps) + 1;
  bp->pages_path = (rows_path >> ps) + 1;
  bp->n_buckets = W * (bp->pages_tok + bp->pages_path);
  return bp->n_buckets <= kMaxBuckets;
}
int sort_entries(c2v_engine* e, cudaStream_t st, const ContextSource& cs, const BucketPlan& bp) {
  PhaseTimer pt(e, PH_PEER_SORT, st);
  int32_t* counts = wsp<int32_t>(e, e->ws.bkt_count);
  int32_t* cursor = wsp<int32_t>(e, e->ws.bkt_cursor);
  if (!e->bkt_zeroed) {
    C2V_CUDA(e, cudaMemsetAsync(counts, 0, (size_t)kMaxBuckets * 4, st));
    e->bkt_zeroed = true;
  }
  const int total = 3 * cs.rows;
  int blocks = (total + 255) / 256;
  if (blocks > e->num_sms * 8) blocks = e->num_sms * 8;
  C2V_LAUNCH(e, (bucket_count_kernel<<<blocks, 256, (size_t)bp.n_buckets * 4, st>>>(cs, bp, counts)));
  C2V_LAUNCH(e, (bucket_scan_kernel<<<1, 1024, 0, st>>>(counts, cursor, wsp<int32_t>(e, e->ws.bkt_starts), bp.n_buckets)));
  C2V_LAUNCH(e, (bucket_fill_kernel<<<blocks, 256, 0, st>>>(cs, bp, cursor, wsp<int32_t>(e, e->ws.perm))));
  return C2V_OK;
}

// Option "deterministic": the sum of each referenced gradient row in the fixed order of DESIGN.md section 5.1 -- a stable radix
// sort of the `count` entries by key (keys in [0, nkeys]; nkeys marks an entry that contributes nothing), then chunk sums and
// their combine.  Every referenced row is stored (the rows are zero before); no atomics, so the result is the same on every run.
// det_sort leaves the sorted keys / entries in ws.det_keys[*cur] / ws.det_vals[*cur]; the other pair is free afterwards.
template <class KeyFn>
int det_sort(c2v_engine* e, cudaStream_t st, const KeyFn& key, int count, uint32_t nkeys, int* cur_out) {
  int bits = 1;
  while (bits < 32 && (1ull << bits) <= nkeys) ++bits;
  uint32_t* keys[2] = {wsp<uint32_t>(e, e->ws.det_keys[0]), wsp<uint32_t>(e, e->ws.det_keys[1])};
  int32_t* vals[2] = {wsp<int32_t>(e, e->ws.det_vals[0]), wsp<int32_t>(e, e->ws.det_vals[1])};
  int32_t* hist = wsp<int32_t>(e, e->ws.det_hist);
  int32_t* offs = wsp<int32_t>(e, e->ws.det_offs);
  int blocks = (count + 255) / 256;
  if (blocks > e->num_sms * 8) blocks = e->num_sms * 8;
  C2V_LAUNCH(e, (det_keys_kernel<KeyFn><<<blocks, 256, 0, st>>>(key, count, keys[0], vals[0])));
  const int tiles = (count + kDetSortTile - 1) / kDetSortTile;
  int cur = 0;
  for (int shift = 0; shift < bits; shift += 8, cur ^= 1) {
    C2V_LAUNCH(e, (det_hist_kernel<<<tiles, kDetSortThreads, 0, st>>>(keys[cur], count, shift, hist)));
    C2V_LAUNCH(e, (bucket_scan_kernel<<<1, 1024, 0, st>>>(hist, offs, wsp<int32_t>(e, e->ws.det_starts), kDetRadix * tiles)));
    C2V_LAUNCH(e, (det_scatter_kernel<<<tiles, kDetSortThreads, 0, st>>>(keys[cur], vals[cur], count, shift, offs, keys[cur ^ 1],
                                                                         vals[cur ^ 1])));
  }
  *cur_out = cur;
  return C2V_OK;
}
template <class Contrib, class Dest>
int det_reduce(c2v_engine* e, cudaStream_t st, int cur, int count, uint32_t nkeys, const Contrib& contrib, const Dest& dst) {
  const uint32_t* keys = wsp<uint32_t>(e, e->ws.det_keys[cur]);
  const unsigned grid = (unsigned)((count + 255) / 256);
  float* part = wsp<float>(e, e->ws.det_part);
  C2V_LAUNCH(e, (det_chunk_kernel<Contrib, Dest><<<grid, 256, 0, st>>>(keys, wsp<int32_t>(e, e->ws.det_vals[cur]), count, nkeys, contrib,
                                                                       dst, part)));
  C2V_LAUNCH(e, (det_combine_kernel<Dest><<<grid, 256, 0, st>>>(keys, count, nkeys, dst, part)));
  return C2V_OK;
}
template <class KeyFn, class Contrib>
int det_row_sums(c2v_engine* e, cudaStream_t st, const KeyFn& key, int count, uint32_t nkeys, const Contrib& contrib,
                 const DetDest& dst) {
  if (count <= 0) return C2V_OK;
  int cur, rc;
  if ((rc = det_sort(e, st, key, count, nkeys, &cur))) return rc;
  return det_reduce(e, st, cur, count, nkeys, contrib, dst);
}

// The embedding-gradient scatter of a train step in deterministic mode, from dX' in dXg.  simt_order: the contributions are
// formed as simt::ScatterDx forms them ((g * m) * s), else as scatter_dx_kernel does (g * (m * s)).
int det_scatter(c2v_engine* e, cudaStream_t st, const ContextSource& cs, const float* mask, const Dropout& dp, const float* dXg,
                bool simt_order) {
  const c2v_dims& d = e->dims;
  const DetStepKeys key{cs.src, cs.pth, cs.tgt, mask, d.token_vocab, (uint32_t)(d.token_vocab + d.path_vocab)};
  const DetDest dst{e->gr_tok.base[0], e->gr_path.base[0], d.token_vocab, d.embed_dim};      // world 1: row r at base[0] + r d
  if (simt_order)
    return det_row_sums(e, st, key, 3 * cs.rows, key.nkeys, DetStepContrib<true>{dXg, dp, e->grad_scale, d.embed_dim}, dst);
  return det_row_sums(e, st, key, 3 * cs.rows, key.nkeys, DetStepContrib<false>{dXg, dp, e->grad_scale, d.embed_dim}, dst);
}

// Option "ordered_exchange" on row-sharded tables: is this engine's embedding-gradient scatter the ordered push?
bool ordered_route(const c2v_engine* e) { return e->ordered_exchange && e->table_world > 1; }

ExchangeKeyMap exchange_key_map(const c2v_engine* e) {
  const int W = e->table_world, Tl = (e->dims.token_vocab + W - 1) / W, Pl = (e->dims.path_vocab + W - 1) / W;
  return ExchangeKeyMap{e->gr_tok.shift, e->gr_tok.mask, Tl, Tl + Pl};
}
// the owner-major keys, W (Tl + Pl) for masked entries included, must sort as 31-bit numbers on any world size
bool exchange_keys_fit(const c2v_dims& d) { return (int64_t)d.token_vocab + d.path_vocab + 2 * kMaxShards < INT32_MAX; }

// The sender's half of the ordered exchange (DESIGN.md section 5.1): one fixed-order sum per distinct (owner, table, row) of
// the `count` entries, stored densely and in key order into this rank's region of each owner's inbox, with the row ids and
// the two counts.  The head ranks live in the sort's spare entry buffer, the per-tile head counts and their scan in its
// histogram buffers, and the 2 W + 1 bounds in ws.det_starts: the workspace is that of option "deterministic".
template <class KeyFn, class Contrib>
int exchange_push(c2v_engine* e, cudaStream_t st, const KeyFn& key, int count, const Contrib& contrib) {
  const ExchangeKeyMap map = exchange_key_map(e);
  const uint32_t nkeys = (uint32_t)e->table_world * map.L;
  int32_t* bounds = wsp<int32_t>(e, e->ws.det_starts);
  e->exchange_pushed = true;
  if (count <= 0) {            // nothing to push: zero counts in every owner's inbox
    C2V_LAUNCH(e, (exchange_bounds_kernel<<<1, 32, 0, st>>>(nullptr, nullptr, 0, map, e->inbox, bounds)));
    return C2V_OK;
  }
  int cur, rc;
  if ((rc = det_sort(e, st, key, count, nkeys, &cur))) return rc;
  const uint32_t* keys = wsp<uint32_t>(e, e->ws.det_keys[cur]);
  int32_t* head_rank = wsp<int32_t>(e, e->ws.det_vals[cur ^ 1]);
  int32_t* tile_heads = wsp<int32_t>(e, e->ws.det_hist);
  int32_t* tile_base = wsp<int32_t>(e, e->ws.det_offs);
  const int tiles = (count + kDetSortTile - 1) / kDetSortTile;
  C2V_LAUNCH(e, (det_head_count_kernel<<<tiles, kDetSortThreads, 0, st>>>(keys, count, nkeys, tile_heads)));
  C2V_LAUNCH(e, (bucket_scan_kernel<<<1, 1024, 0, st>>>(tile_heads, tile_base, bounds, tiles)));
  C2V_LAUNCH(e, (det_head_rank_kernel<<<tiles, kDetSortThreads, 0, st>>>(keys, count, nkeys, tile_base, head_rank)));
  C2V_LAUNCH(e, (exchange_bounds_kernel<<<1, 32, 0, st>>>(keys, head_rank, count, map, e->inbox, bounds)));
  const DetInboxDest dst{e->inbox, head_rank, bounds, map.L, e->dims.embed_dim};
  C2V_LAUNCH(e, (exchange_ids_kernel<<<(count + 255) / 256, 256, 0, st>>>(keys, count, map, dst)));
  return det_reduce(e, st, cur, count, nkeys, contrib, dst);
}

// The embedding-gradient scatter of a train step on row-sharded tables under option "ordered_exchange", from dX' in dXg
int exchange_scatter(c2v_engine* e, cudaStream_t st, const ContextSource& cs, const float* mask, const Dropout& dp, const float* dXg,
                     bool simt_order) {
  const int d = e->dims.embed_dim;
  const ExchangeStepKeys key{cs.src, cs.pth, cs.tgt, mask, exchange_key_map(e)};
  if (simt_order) return exchange_push(e, st, key, 3 * cs.rows, DetStepContrib<true>{dXg, dp, e->grad_scale, d});
  return exchange_push(e, st, key, 3 * cs.rows, DetStepContrib<false>{dXg, dp, e->grad_scale, d});
}

// Grid of the gather: one wave of resident CTAs (8 warps each; a warp strides over the rows), never more CTAs than rows / 8.
unsigned gather_blocks(c2v_engine* e, int rows, bool split) {
  int& occ = e->gather_occ[split ? 1 : 0];
  if (occ == 0) {
    int n = 0;
    cudaError_t rc = split ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, gather_ctx_kernel<true>, 256, 0)
                           : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, gather_ctx_kernel<false>, 256, 0);
    occ = (rc == cudaSuccess && n > 0) ? n : 4;
  }
  const long want = (rows + 7) / 8, wave = (long)e->num_sms * occ;
  return (unsigned)(want < wave ? want : wave);
}

// H = tanh(X' . W)   (tensorflow_model.py:238-252)
int run_ctx_fwd(c2v_engine* e, cudaStream_t st, const ContextSource& cs, const Dropout& dp, float* H, bool keep_x) {
  const int D = e->dims.code_dim, K = 3 * e->dims.embed_dim;
  { int rc0 = prepare_rows(e, st, cs); if (rc0) return rc0; }
  if (is_tc(e) && !is_3x(e) && e->fuse_gather && e->dims.embed_dim % 32 == 0 && cs.rows % 4 == 0 &&
      (((uintptr_t)cs.src | (uintptr_t)cs.pth | (uintptr_t)cs.tgt) % 16) == 0) {
    // gather -> dropout -> projection -> tanh in one kernel (umma::launch_ctx_fused); X' is written out only when a backward
    // pass will need it (dW = X'^T . dU)
    PhaseTimer pt(e, PH_CTX_FWD, st);
    umma::EpiTanhStore ep{H, (size_t)D};
    C2V_LAUNCH(e, C2V_CUDA(e, (umma::launch_ctx_fused(st, cs.rows, D, e->theta.W, (size_t)D, cs, dp,
                                                              keep_x ? wsp<float>(e, e->ws.Xg) : nullptr, ep, e->num_sms))));
    return C2V_OK;
  }
  if (is_tc(e)) {
    float* Xg = wsp<float>(e, e->ws.Xg);
    const bool x3 = is_3x(e);
    {
      PhaseTimer pt(e, PH_GATHER, st);
      BucketPlan bp;
      e->sorted_src = nullptr;
      if (e->inbox.world > 1 && !ordered_route(e) && plan_buckets(e, &bp, true) && !plan_buckets(e, &bp)) {
        // the backward pass will push gradient rows owner by owner: bucket the batch now, while the SMs are free (in
        // the backward pass the same three small kernels would queue behind the persistent dW GEMM)
        int rcs = sort_entries(e, st, cs, bp);
        if (rcs) return rcs;
        e->sorted_src = cs.src; e->sorted_rows = cs.rows;
      }
      if (plan_buckets(e, &bp)) {           // peer shards: walk the entries page by page
        int rcs = sort_entries(e, st, cs, bp);
        if (rcs) return rcs;
        e->sorted_src = cs.src; e->sorted_rows = cs.rows;
        const int32_t* perm = wsp<int32_t>(e, e->ws.perm);
        if (x3) C2V_LAUNCH(e, (gather_sorted_kernel<true><<<(3 * cs.rows + 7) / 8, 256, 0, st>>>(cs, dp, perm, Xg, wsp<float>(e, e->ws.Xg_lo))));
        else C2V_LAUNCH(e, (gather_sorted_kernel<false><<<(3 * cs.rows + 7) / 8, 256, 0, st>>>(cs, dp, perm, Xg, nullptr)));
      } else if (x3) C2V_LAUNCH(e, (gather_ctx_kernel<true><<<gather_blocks(e, cs.rows, true), 256, 0, st>>>(cs, dp, Xg, wsp<float>(e, e->ws.Xg_lo))));
      else C2V_LAUNCH(e, (gather_ctx_kernel<false><<<gather_blocks(e, cs.rows, false), 256, 0, st>>>(cs, dp, Xg, nullptr)));
    }
    // B = W^T, K-major.  3xTF32: one pass writes its split and the split of W itself, which dx_gemm reads
    if (x3) {
      PhaseTimer pt(e, PH_SPLIT, st);
      int rcs = transpose_operand(e, st, e->theta.W, K, D, (size_t)K, e->ws.WT, true, e->ws.WT_lo, wsp<float>(e, e->ws.W_hi),
                                  wsp<float>(e, e->ws.W_lo));
      if (rcs) return rcs;
    }
    PhaseTimer pt(e, PH_CTX_FWD, st);
    if (!x3) { int rcs = transpose_operand(e, st, e->theta.W, K, D, (size_t)K, e->ws.WT, false); if (rcs) return rcs; }
    umma::Operand opA{Xg, (size_t)K, false, x3 ? wsp<float>(e, e->ws.Xg_lo) : nullptr};
    umma::Operand opB{wsp<float>(e, e->ws.WT), (size_t)K, false, x3 ? wsp<float>(e, e->ws.WT_lo) : nullptr};
    if (x3) {
      umma::EpiTanhStorePrecise ep{H, (size_t)D};
      C2V_LAUNCH(e, C2V_CUDA(e, (umma::launch_cfg<false, false, umma::EpiTanhStorePrecise>(st, cs.rows, D, K, 1, opA, opB, ep, e->num_sms))));
    } else {
      umma::EpiTanhStore ep{H, (size_t)D};
      C2V_LAUNCH(e, C2V_CUDA(e, (umma::launch_cfg<false, false, umma::EpiTanhStore>(st, cs.rows, D, K, 1, opA, opB, ep, e->num_sms))));
    }
    return C2V_OK;
  }
  PhaseTimer pt(e, PH_CTX_FWD, st);
  simt::GatherRowsK al{cs, dp};
  simt::ColsX bl{e->theta.W, (size_t)D};
  simt::TanhStore ep{H, (size_t)D};
  C2V_LAUNCH(e, C2V_CUDA(e, simt::launch(st, cs.rows, D, K, 1, al, bl, ep)));
  return C2V_OK;
}

// What the logits GEMM S[B, Y] = v . Ytab^T (tensorflow_model.py:226,297) leaves in ws.S; "partials" are the per-(row,
// partial slot) (max, sum exp) pairs (umma::lse_slots) it also writes to ws.lse_part
enum LogitsOut {
  LOGITS_STORE,            // the logits
  LOGITS_STORE_LSE,        // the logits and their partials
  LOGITS_LSE_ONLY,         // the partials only
  LOGITS_SOFTMAX_GRAD,     // dL/dlogits = (softmax - onehot) * inv_batch, from the log-sum-exp in LogitsArgs::sg
  LOGITS_EXP_SUM,          // U = exp(s - LogitsArgs::exp_offset[row]) and (max U, sum U) partials
  LOGITS_STORE_LSE_GATED,  // as LOGITS_STORE_LSE while *LogitsArgs::gate != 0, else nothing (the exp_slab fallback)
  LOGITS_TOPK,             // nothing: each (row, partial slot)'s best LogitsArgs::topk_k candidates (topk_candidates)
  LOGITS_TOPK_LSE,         // the candidates and the partials
};
struct LogitsArgs {
  const float* exp_offset;
  const int* gate;
  umma::SoftmaxGradArgs sg;
  int topk_k;
  int row0;                // first global class of this engine's table (candidate ids)
};

// Candidate lists of the top-k epilogue in ws.S: values [B, lse_slots(Y), k], then the ids.  For k <= kTopkEpiMax that is
// 2 x 4 x 16 x 2 ceil(Y / 128) <= 4 ldS bytes per row: the slab region holds them, and the workspace is unchanged.
struct TopkCandidates {
  float* val;
  int32_t* idx;
};
inline TopkCandidates topk_candidates(c2v_engine* e, int B, int k) {
  float* S = wsp<float>(e, e->ws.S);
  return {S, reinterpret_cast<int32_t*>(S + (size_t)B * umma::lse_slots(e->dims.target_vocab) * k)};
}

// for_dv: a dv GEMM of this step follows, so the GEMM also writes Ytab^T (3xTF32: its transposed split) from the Ytab tiles it
// streams, from the same table (umma::BTransposed).  Only the first logits pass of a step, whose epilogues take go_dv, does.
template <bool X3>
int launch_logits(c2v_engine* e, cudaStream_t st, const float* v, int B, LogitsOut out, const LogitsArgs& a, bool for_dv) {
  const int D = e->dims.code_dim, Y = e->dims.target_vocab;
  umma::Operand opA{v, (size_t)D, false};
  umma::Operand opB{e->theta.tgt, (size_t)D, false};
  int rcs;
  if (X3) {      // fp32-faithful: both operands as tf32 (hi, lo) pairs; the gated fallback reuses the previous pass's splits
    if (out != LOGITS_STORE_LSE_GATED) {
      if ((rcs = split_small(e, st, v, (size_t)B * D, e->ws.v_hi, e->ws.v_lo))) return rcs;
      if ((rcs = split_small(e, st, e->theta.tgt, (size_t)Y * D, e->ws.tgt_hi, e->ws.tgt_lo))) return rcs;
    }
    opA.base = wsp<float>(e, e->ws.v_hi); opA.lo = wsp<float>(e, e->ws.v_lo);
    opB.base = wsp<float>(e, e->ws.tgt_hi); opB.lo = wsp<float>(e, e->ws.tgt_lo);
  }
  PhaseTimer pt(e, PH_LOGITS, st);
  float* S = wsp<float>(e, e->ws.S);
  float* S_lo = X3 ? wsp<float>(e, e->ws.S_lo) : nullptr;
  const size_t ld = e->ws.ldS;
  const umma::EpiStoreLseT<X3> lse{S, ld, wsp<float2>(e, e->ws.lse_part), umma::lse_slots(Y)};
  auto go = [&](auto ep) -> int {
    C2V_LAUNCH(e, C2V_CUDA(e, (umma::launch_cfg<false, false, decltype(ep)>(st, B, Y, D, 1, opA, opB, ep, e->num_sms))));
    return C2V_OK;
  };
  auto go_dv = [&](auto ep) -> int {
    if (!for_dv) return go(ep);
    const umma::BTransposed bt{wsp<float>(e, e->ws.tgtT), X3 ? wsp<float>(e, e->ws.tgtT_lo) : nullptr, e->ws.ldS};
    C2V_LAUNCH(e, C2V_CUDA(e, (umma::launch_cfg<false, false, decltype(ep), umma::AXNone, true>(st, B, Y, D, 1, opA, opB, ep, e->num_sms,
                                                                                                umma::AXNone{}, bt))));
    e->tgt_t_valid = true;
    return C2V_OK;
  };
  switch (out) {
    case LOGITS_STORE: return go_dv(umma::EpiStore{S, ld, 0});
    case LOGITS_STORE_LSE: return go_dv(lse);
    case LOGITS_LSE_ONLY: return go_dv(umma::EpiLseOnlyT<X3>{lse});
    case LOGITS_SOFTMAX_GRAD:
      return go(umma::EpiSoftmaxGradT<X3, X3>{S, S_lo, ld, a.sg.lse, a.sg.target, a.sg.row0, a.sg.inv_batch, B});
    case LOGITS_EXP_SUM: return go_dv(umma::EpiExpSumT<X3, X3>{S, S_lo, ld, a.exp_offset, lse.partial, lse.slots});
    case LOGITS_STORE_LSE_GATED: return go(umma::EpiStoreLseGatedT<X3>{lse, a.gate});
    case LOGITS_TOPK:
    case LOGITS_TOPK_LSE: {
      const TopkCandidates c = topk_candidates(e, B, a.topk_k);
      if (out == LOGITS_TOPK_LSE) return go(umma::EpiTopkT<X3, true>{lse, c.val, c.idx, a.topk_k, a.row0});
      return go(umma::EpiTopkT<X3, false>{lse, c.val, c.idx, a.topk_k, a.row0});
    }
  }
  return C2V_OK;
}

int run_logits(c2v_engine* e, cudaStream_t st, const float* v, int B, LogitsOut out, const LogitsArgs& a = {}, bool for_dv = false) {
  { int rcl = end_target_lazy(e, st); if (rcl) return rcl; }      // a pass over the whole table needs every row current
  if (is_tc(e) && aligned16(v))
    return is_3x(e) ? launch_logits<true>(e, st, v, B, out, a, for_dv) : launch_logits<false>(e, st, v, B, out, a, for_dv);
  const int D = e->dims.code_dim;
  PhaseTimer pt(e, PH_LOGITS, st);
  if (!aligned16(v)) {        // the SIMT loaders read float4s: code vectors a caller passed unaligned go through a copy
    float* va = wsp<float>(e, e->ws.v_scaled);
    if (e->pending_dy.v == va) return fail(e, C2V_ERR_STATE, "a deferred dY still reads the exp_slab scaled code vectors");
    C2V_CUDA(e, cudaMemcpyAsync(va, v, (size_t)B * D * 4, cudaMemcpyDeviceToDevice, st));
    v = va;
  }
  simt::RowsK al{v, (size_t)D};
  simt::RowsK bl{e->theta.tgt, (size_t)D};
  simt::StoreC ep{wsp<float>(e, e->ws.S), e->ws.ldS, 0};
  C2V_LAUNCH(e, C2V_CUDA(e, simt::launch(st, B, e->dims.target_vocab, D, 1, al, bl, ep)));
  return C2V_OK;
}

int forward_impl(c2v_engine* e, cudaStream_t st, const int32_t* src, const int32_t* pth, const int32_t* tgt,
                 const float* mask, int B, const Dropout& dp, float* code_vec, float* attn, bool keep_x = false) {
  ContextSource cs = make_source(e, src, pth, tgt, B);
  float* H = wsp<float>(e, e->ws.H);
  int rc = run_ctx_fwd(e, st, cs, dp, H, keep_x);
  if (rc) return rc;
  if ((rc = launch_attn_fwd(e, st, H, mask, B, attn, code_vec))) return rc;
  if (keep_x && code_vec != wsp<float>(e, e->ws.v))      // a backward pass follows (phase-split API): it needs the code vectors
    C2V_CUDA(e, cudaMemcpyAsync(wsp<float>(e, e->ws.v), code_vec, (size_t)B * e->dims.code_dim * 4, cudaMemcpyDeviceToDevice, st));
  return C2V_OK;
}

int topk_impl(c2v_engine* e, cudaStream_t st, const float* code_vec, int B, int32_t* idx, float* val, int normalize) {
  if (normalize < 0 || normalize > 2) return fail(e, C2V_ERR_INVALID, "normalize must be 0 (logits), 1 (softmax over k) or 2 (full softmax)");
  float* S = wsp<float>(e, e->ws.S);
  int rc = run_logits(e, st, code_vec, B, LOGITS_STORE);
  if (rc) return rc;
  const int Y = e->dims.target_vocab;
  const int k = e->dims.top_k < Y ? e->dims.top_k : Y;
  PhaseTimer pt(e, PH_TOPK, st);
  if (k <= 16)
    C2V_LAUNCH(e, (topk_kernel<16><<<B, kTopkThreads, 0, st>>>(S, e->ws.ldS, Y, k, normalize, idx, val)));
  else
    C2V_LAUNCH(e, (topk_iter_kernel<<<B, kTopkThreads, 0, st>>>(S, e->ws.ldS, Y, k, normalize, idx, val)));
  if (normalize == 2) C2V_LAUNCH(e, (topk_full_softmax_kernel<<<B, 256, 0, st>>>(S, e->ws.ldS, Y, k, val)));
  return C2V_OK;
}

// This engine's best k rows (global ids row0 + local row) per example, raw logits, padded with (-inf, INT_MAX); with row_max /
// row_sum, the (max, sum exp) of each example's logits over the local rows.  Tensor cores and k <= kTopkEpiMax: the logits
// epilogue keeps per-(row, slot) candidate lists and topk_merge_kernel merges a row's slots, so no logit is stored.  fp32
// (SIMT logits) and larger k: the logits slab, scanned by the kernels of c2v_topk.
int topk_partial_impl(c2v_engine* e, cudaStream_t st, const float* code_all, int Bt, int row0, int k, int32_t* idx, float* val,
                      float* row_max, float* row_sum) {
  const int Y = e->dims.target_vocab;
  const int slots = umma::lse_slots(Y);
  float* S = wsp<float>(e, e->ws.S);
  float2* part = wsp<float2>(e, e->ws.lse_part);
  const bool stats = row_max != nullptr;
  int rc;
  if (is_tc(e) && aligned16(code_all) && k <= umma::kTopkEpiMax) {
    LogitsArgs la{};
    la.topk_k = k;
    la.row0 = row0;
    if ((rc = run_logits(e, st, code_all, Bt, stats ? LOGITS_TOPK_LSE : LOGITS_TOPK, la))) return rc;
    PhaseTimer pt(e, PH_TOPK, st);
    const TopkCandidates c = topk_candidates(e, Bt, k);
    const TopkMergeArgs ma{c.idx, c.val, slots, (size_t)slots * k, (size_t)k, k, 0, nullptr, nullptr, 1, Bt, 0, idx, val};
    C2V_LAUNCH(e, (topk_merge_kernel<umma::kTopkEpiMax><<<Bt, kTopkThreads, 0, st>>>(ma)));
    if (stats) C2V_LAUNCH(e, (row_maxsum_kernel<<<Bt, 256, 0, st>>>(part, slots, S, e->ws.ldS, Y, nullptr, 0, row_max, row_sum, nullptr)));
    return C2V_OK;
  }
  if ((rc = run_logits(e, st, code_all, Bt, LOGITS_STORE))) return rc;
  PhaseTimer pt(e, PH_TOPK, st);
  if (k <= 16)
    C2V_LAUNCH(e, (topk_kernel<16><<<Bt, kTopkThreads, 0, st>>>(S, e->ws.ldS, Y, k, 0, idx, val, row0)));
  else
    C2V_LAUNCH(e, (topk_iter_kernel<<<Bt, kTopkThreads, 0, st>>>(S, e->ws.ldS, Y, k, 0, idx, val, row0)));
  if (stats) C2V_LAUNCH(e, (row_maxsum_kernel<<<Bt, 256, 0, st>>>(nullptr, 0, S, e->ws.ldS, Y, nullptr, 0, row_max, row_sum, nullptr)));
  return C2V_OK;
}

int run_dy(c2v_engine* e, cudaStream_t st, const float* v, int B, const SlabDesc& slab);

// the dY product target_grad_gemms deferred, if any
int run_pending_dy(c2v_engine* e, cudaStream_t st) {
  if (!e->pending_dy.v) return C2V_OK;
  const PendingDy p = e->pending_dy;
  e->pending_dy = PendingDy{};
  return run_dy(e, st, p.v, p.B, p.slab);
}

// Backward of everything below the code vector, given dv: gradients of a, W and the two
// embedding tables (SURVEY A.2).
int context_backward(c2v_engine* e, cudaStream_t st, const ContextSource& cs, const float* mask, int B,
                     const Dropout& dp, const float* dv) {
  const int D = e->dims.code_dim, d = e->dims.embed_dim, K3 = 3 * d, N = cs.rows;
  float* H = wsp<float>(e, e->ws.H);
  float* alpha = wsp<float>(e, e->ws.alpha);
  float* da_part = wsp<float>(e, e->ws.da_part);
  float* part = wsp<float>(e, e->ws.part);
  int rc;
  if (ordered_route(e) && e->inbox.world < 2)
    return fail(e, C2V_ERR_STATE, "ordered_exchange: the gradient rows of row-sharded tables travel through the scatter inbox, "
                                  "and none is bound (c2v_bind_scatter_inbox)");
  if (!is_tc(e) && (rc = run_pending_dy(e, st))) return rc;     // fp32 path: nothing to overlap with, run it first
  const bool x3 = is_tc(e) && is_3x(e);
  float* H_lo = x3 ? wsp<float>(e, e->ws.H_lo) : nullptr;
  rc = launch_attn_bwd(e, st, H, alpha, dv, wsp<float>(e, e->ws.v), B, da_part, H_lo);    // H now holds dU (3xTF32: its high parts, H_lo the rest)
  if (rc) return rc;
  rc = launch_colsum(e, st, da_part, (size_t)D, B, D, e->grad.a);
  if (rc) return rc;
  if (is_tc(e)) {
    float* Xg = wsp<float>(e, e->ws.Xg);
    float* dXg = wsp<float>(e, e->ws.dXg);
    {  // dX' = dU . W^T
      PhaseTimer pt(e, PH_DX_GEMM, st);
      // 3xTF32: W's split was made by this step's forward pass (run_ctx_fwd) and W has not changed since
      umma::Operand opA{H, (size_t)D, false, H_lo};
      umma::Operand opB{x3 ? wsp<float>(e, e->ws.W_hi) : e->theta.W, (size_t)D, false, x3 ? wsp<float>(e, e->ws.W_lo) : nullptr};
      umma::EpiStore ep{dXg, (size_t)K3, 0};
      C2V_LAUNCH(e, C2V_CUDA(e, (umma::launch(st, N, K3, D, 1, opA, opB, ep, e->num_sms))));
    }
    if (e->lazy) {
      if (e->lazy_grads_pending)
        return fail(e, C2V_ERR_STATE, "lazy_adam: every train step must be followed by c2v_adam_step before the next one");
      e->lazy_grads_pending = true;
    } else if (!e->emb_grads_clean && e->table_world == 1) {
      C2V_CUDA(e, cudaMemsetAsync(e->grad.tok, 0, (size_t)e->dims.token_vocab * d * 4, st));
      C2V_CUDA(e, cudaMemsetAsync(e->grad.path, 0, (size_t)e->dims.path_vocab * d * 4, st));
    }
    // fork: the scatter-add of dX' rows (memory / NVLink bound, no shared memory) runs on the engine's
    // side stream while the dW GEMM (tensor bound) runs on the caller's stream; join before returning.
    C2V_CUDA(e, cudaEventRecord(e->ev_fork, st));
    C2V_CUDA(e, cudaStreamWaitEvent(e->side, e->ev_fork, 0));
    {
      PhaseTimer pt(e, PH_DX_SCATTER, e->side);
      BucketPlan bp;
      if (ordered_route(e)) {      // one fixed-order sum per distinct row into the owner's inbox; the owners fold in rank order
        e->sorted_src = nullptr;
        if ((rc = exchange_scatter(e, e->side, cs, mask, dp, dXg, false))) return rc;
      } else if (e->inbox.world > 1 && plan_buckets(e, &bp, true)) {
        // push: every owner's rows go densely into this rank's region of the owner's inbox (plain coalesced stores over
        // NVLink); the owners fold them in with local atomics after the caller's barrier (c2v_apply_scatter_inbox)
        if (e->sorted_src != cs.src || e->sorted_rows != cs.rows) {     // not bucketed by this step's forward pass
          if ((rc = sort_entries(e, e->side, cs, bp))) return rc;
        }
        e->sorted_src = nullptr;
        const int32_t* starts = wsp<int32_t>(e, e->ws.bkt_starts);
        C2V_LAUNCH(e, (inbox_counts_kernel<<<1, 32, 0, e->side>>>(e->inbox, bp, starts)));
        C2V_LAUNCH(e, (scatter_inbox_kernel<<<(3 * N + 7) / 8, 256, 0, e->side>>>(cs, dp, mask, wsp<int32_t>(e, e->ws.perm), starts, bp, dXg,
                                                                              e->inbox, e->grad_scale)));
      } else if (plan_buckets(e, &bp)) {    // peer shards: the red.adds walk the owners' pages in order
        if ((rc = sort_entries(e, e->side, cs, bp))) return rc;
        C2V_LAUNCH(e, (scatter_sorted_kernel<<<(3 * N + 7) / 8, 256, 0, e->side>>>(cs, dp, mask, wsp<int32_t>(e, e->ws.perm), dXg, e->gr_tok,
                                                                               e->gr_path, e->grad_scale)));
      } else if (e->deterministic) {      // sorted, fixed-order row sums instead of float atomics
        if ((rc = det_scatter(e, e->side, cs, mask, dp, dXg, false))) return rc;
      } else {
        C2V_LAUNCH(e, (scatter_dx_kernel<<<(N + 7) / 8, 256, 0, e->side>>>(cs, dp, mask, dXg, e->gr_tok, e->gr_path, e->grad_scale)));
      }
    }
    if ((rc = early_catchup(e, e->side))) return rc;
    C2V_CUDA(e, cudaEventRecord(e->ev_join, e->side));
    if ((rc = run_pending_dy(e, st))) return rc;     // concurrent with the scatter-add
    {  // dW = X'^T . dU on the gathered X' kept from the forward pass
      PhaseTimer pt(e, PH_DW, st);
      umma::Operand opA{Xg, (size_t)K3, true, x3 ? wsp<float>(e, e->ws.Xg_lo) : nullptr};
      umma::Operand opB{H, (size_t)D, true, H_lo};
      const int ks = umma::effective_splits(N, kSplitDw);
      umma::EpiStore ep{part, (size_t)D, (size_t)K3 * D};
      C2V_LAUNCH(e, C2V_CUDA(e, (umma::launch(st, K3, D, N, kSplitDw, opA, opB, ep, e->num_sms))));
      rc = launch_colsum(e, st, part, (size_t)K3 * D, ks, K3 * D, e->grad.W);
      if (rc) return rc;
    }
    C2V_CUDA(e, cudaStreamWaitEvent(st, e->ev_join, 0));
    if (e->dy_in_flight) {
      C2V_CUDA(e, cudaStreamWaitEvent(st, e->ev_join2, 0));
      e->dy_in_flight = false;
    }
    e->emb_grads_clean = false;
    return C2V_OK;
  }
  {  // dW = X'^T . dU   (split-K over the B*C contexts, fixed-order reduction)
    PhaseTimer pt(e, PH_DW, st);
    simt::GatherColsX al{cs, dp};
    simt::ColsX bl{H, (size_t)D};
    const int ks = simt::effective_ksplit(N, kSplitDw);
    simt::StoreC ep{part, (size_t)D, (size_t)K3 * D};
    C2V_LAUNCH(e, C2V_CUDA(e, simt::launch(st, K3, D, N, kSplitDw, al, bl, ep)));
    rc = launch_colsum(e, st, part, (size_t)K3 * D, ks, K3 * D, e->grad.W);
    if (rc) return rc;
  }
  {  // dX' = dU . W^T -> dropout backward -> scatter-add into the embedding gradient tables
    if (e->lazy) {
      if (e->lazy_grads_pending)
        return fail(e, C2V_ERR_STATE, "lazy_adam: every train step must be followed by c2v_adam_step before the next one");
      e->lazy_grads_pending = true;
    } else if (!e->emb_grads_clean && e->table_world == 1) {
      C2V_CUDA(e, cudaMemsetAsync(e->grad.tok, 0, (size_t)e->dims.token_vocab * d * 4, st));
      C2V_CUDA(e, cudaMemsetAsync(e->grad.path, 0, (size_t)e->dims.path_vocab * d * 4, st));
    }
    PhaseTimer pt(e, PH_DX_SCATTER, st);
    simt::RowsK al{H, (size_t)D};
    simt::RowsK bl{e->theta.W, (size_t)D};
    if (e->deterministic || ordered_route(e)) {        // dX' is stored, then summed row by row in a fixed order
      float* dXg = wsp<float>(e, e->ws.dXg);
      simt::StoreC ep{dXg, (size_t)K3, 0};
      C2V_LAUNCH(e, C2V_CUDA(e, simt::launch(st, N, K3, D, 1, al, bl, ep)));
      if ((rc = ordered_route(e) ? exchange_scatter(e, st, cs, mask, dp, dXg, true) : det_scatter(e, st, cs, mask, dp, dXg, true)))
        return rc;
    } else {
      simt::ScatterDx ep{cs, e->gr_tok, e->gr_path, mask, dp, e->grad_scale};
      C2V_LAUNCH(e, C2V_CUDA(e, simt::launch(st, N, K3, D, 1, al, bl, ep)));
    }
    e->emb_grads_clean = false;
  }
  return C2V_OK;
}

// Given P = dL/dlogits in the S slab (as `slab` describes it):  dv = P . Ytab  (split-K over |Y|, fixed-order reduction).
int run_dv(c2v_engine* e, cudaStream_t st, int B, float* dv, const SlabDesc& slab) {
  const int D = e->dims.code_dim, Y = e->dims.target_vocab;
  float* S = wsp<float>(e, e->ws.S);
  float* part = wsp<float>(e, e->ws.part);
  PhaseTimer pt(e, PH_DV, st);
  if (is_tc(e)) {
    // B = Ytab^T, K-major, made by this step's logits pass (3xTF32: as the table's split; P was written as its split by
    // softmax_grad_kernel)
    if (!e->tgt_t_valid) { int rct = transpose_table(e, st); if (rct) return rct; }
    umma::Operand opA{S, e->ws.ldS, false};
    umma::Operand opB{wsp<float>(e, e->ws.tgtT), e->ws.ldS, false};
    if (is_3x(e)) {
      opA.lo = wsp<float>(e, e->ws.S_lo);
      opB.lo = wsp<float>(e, e->ws.tgtT_lo);
    }
    // enough split-K slices to fill the SMs about twice; few when the batch already gives many tiles
    const int tiles = ((B + umma::BM - 1) / umma::BM) * ((D + umma::BN - 1) / umma::BN);
    int want = (2 * e->num_sms + tiles - 1) / tiles;
    if (want > kSplitDv) want = kSplitDv;
    const int ks = umma::effective_splits(Y, want);
    umma::EpiStore ep{part, (size_t)D, (size_t)B * D};
    if (slab.loaders) {       // A = the logits slab, turned into dL/dlogits by the GEMM's loaders
      umma::AXSoftmaxGrad<true> ax{slab.sg};
      C2V_LAUNCH(e, C2V_CUDA(e, (umma::launch_cfg<false, false, umma::EpiStore, umma::AXSoftmaxGrad<true>>(st, B, D, Y, want, opA, opB, ep,
                                                                                                            e->num_sms, ax))));
    } else {
      C2V_LAUNCH(e, C2V_CUDA(e, (umma::launch(st, B, D, Y, want, opA, opB, ep, e->num_sms))));
    }
    return launch_colsum(e, st, part, (size_t)B * D, ks, B * D, dv, slab.row_scale, D);
  }
  simt::RowsK al{S, e->ws.ldS};
  simt::ColsX bl{e->theta.tgt, (size_t)D};
  const int ks = simt::effective_ksplit(Y, kSplitDv);
  simt::StoreC ep{part, (size_t)D, (size_t)B * D};
  C2V_LAUNCH(e, C2V_CUDA(e, simt::launch(st, B, D, Y, kSplitDv, al, bl, ep)));
  return launch_colsum(e, st, part, (size_t)B * D, ks, B * D, dv);
}

// dYtab = P^T . v  into the bound target-table gradient; then the caller's "target_grads_ready" event.
int run_dy(c2v_engine* e, cudaStream_t st, const float* v, int B, const SlabDesc& slab) {
  const int D = e->dims.code_dim, Y = e->dims.target_vocab;
  float* S = wsp<float>(e, e->ws.S);
  {
    PhaseTimer pt(e, PH_DY, st);
    if (is_3x(e) && !aligned16(v))
      return fail(e, C2V_ERR_INVALID, "3xTF32: the code vectors must be 16-byte aligned");
    if (is_tc(e) && aligned16(v)) {
      // A = S^T stays MN-major (a transposed copy of the slab would cost a write of its own size); B = v^T, K-major
      const size_t ldB = align_up((size_t)B, 4);
      int rcs;
      if (is_3x(e)) {
        PhaseTimer pts(e, PH_SPLIT, st);
        rcs = transpose_operand(e, st, v, B, D, ldB, e->ws.vT, true, e->ws.vT_lo);
      } else {
        rcs = transpose_operand(e, st, v, B, D, ldB, e->ws.vT, false);
      }
      if (rcs) return rcs;
      umma::Operand opA{S, e->ws.ldS, true, is_3x(e) ? wsp<float>(e, e->ws.S_lo) : nullptr};
      umma::Operand opB{wsp<float>(e, e->ws.vT), ldB, false, is_3x(e) ? wsp<float>(e, e->ws.vT_lo) : nullptr};
      auto go = [&](auto ep) -> int {
        if (slab.loaders)       // A = the logits slab, turned into dL/dlogits by the GEMM's loaders
          C2V_LAUNCH(e, C2V_CUDA(e, (umma::launch_cfg<true, false, decltype(ep), umma::AXSoftmaxGrad<false>>(
                                        st, Y, D, B, 1, opA, opB, ep, e->num_sms, umma::AXSoftmaxGrad<false>{slab.sg}))));
        else
          C2V_LAUNCH(e, C2V_CUDA(e, (umma::launch_cfg<true, false, decltype(ep)>(st, Y, D, B, 1, opA, opB, ep, e->num_sms))));
        return C2V_OK;
      };
      int rc;
      if (e->tgt_armed && e->has_adam) {
        // dYtab never reaches memory: the epilogue applies TF1 Adam to the target table in place
        const double lr_t = (double)e->tgt_lr * sqrt(1.0 - pow((double)e->tgt_b2, (double)e->tgt_t)) /
                            (1.0 - pow((double)e->tgt_b1, (double)e->tgt_t));
        if ((rc = go(umma::EpiAdam{e->theta.tgt, e->am.tgt, e->av.tgt, (size_t)D, (float)lr_t, e->tgt_b1, e->tgt_b2, e->tgt_eps,
                                   1.f - e->tgt_b1, 1.f - e->tgt_b2, e->adam_epi_prefetch})))
          return rc;
        e->tgt_armed = false;
        e->tgt_fused_t = e->tgt_t;
        e->tgt_t_valid = false;
      } else if ((rc = go(umma::EpiStore{e->grad.tgt, (size_t)D, 0}))) {
        return rc;
      }
    } else {
      simt::ColsX al{S, e->ws.ldS};
      simt::ColsX bl{v, (size_t)D};
      simt::StoreC ep{e->grad.tgt, (size_t)D, 0};
      C2V_LAUNCH(e, C2V_CUDA(e, simt::launch(st, Y, D, B, 1, al, bl, ep)));
    }
  }
  if (e->ev_tgt_ready) C2V_CUDA(e, cudaEventRecord(e->ev_tgt_ready, st));
  return C2V_OK;
}

// The two target-table gradient products.  With option "dy_late" (default) only dv runs here and dY is
// deferred into context_backward, where it overlaps the NVLink / L2-atomic bound scatter-add of the
// embedding gradients (dY needs P and v only, not the context backward).
int target_grad_gemms(c2v_engine* e, cudaStream_t st, const float* v, int B, float* dv, const SlabDesc& slab) {
  int rc = run_dv(e, st, B, dv, slab);
  if (rc) return rc;
  if (e->dy_late == 2 && is_tc(e)) {
    // dY (and the target table's Adam step in its epilogue) is HBM-bound and independent of the context
    // backward pass: it runs on its own stream from here until context_backward joins it
    C2V_CUDA(e, cudaEventRecord(e->ev_fork2, st));
    C2V_CUDA(e, cudaStreamWaitEvent(e->side2, e->ev_fork2, 0));
    if ((rc = run_dy(e, e->side2, v, B, slab))) return rc;
    C2V_CUDA(e, cudaEventRecord(e->ev_join2, e->side2));
    e->dy_in_flight = true;
    return C2V_OK;
  }
  if (e->dy_late) {
    e->pending_dy = PendingDy{v, B, slab};
    return C2V_OK;
  }
  return run_dy(e, st, v, B, slab);
}

// Turns the slab into P = dL/dlogits = (softmax - onehot) * inv_batch for the dv / dY GEMMs, inside the caller's PH_XENT
// timer; returns in `slab` how they read it, and in `v_dy` the code vectors dY multiplies.  Two-pass: softmax_grad_kernel
// rewrites the logits (3xTF32: as P's split).  Loaders: nothing runs here, the GEMMs' A loaders do it.  exp_slab: the slab
// holds U, already patched; the same rewrite runs gated, for rows that left the fp32 window only (reset_factors: it also
// sets their factors to 1 and counts the fallback), and dY gets the code vectors scaled by the rows' factors.
int slab_to_p(c2v_engine* e, cudaStream_t st, HeadSchedule hs, const float* v, int B, const umma::SoftmaxGradArgs& g,
              SlabDesc* slab, const float** v_dy, bool reset_factors = false) {
  *v_dy = v;
  if (hs == HEAD_LOADERS) {
    slab->loaders = true;
    slab->sg = g;
    return C2V_OK;
  }
  float* S = wsp<float>(e, e->ws.S);
  const int Y = e->dims.target_vocab, D = e->dims.code_dim;
  const bool gated = hs == HEAD_EXP_SLAB;
  const int* gate = gated ? wsp<int>(e, e->ws.slab_flag) : nullptr;
  float* rscale = wsp<float>(e, e->ws.rscale);
  float* reset = gated && reset_factors ? rscale : nullptr;
  unsigned* count = reset ? reinterpret_cast<unsigned*>(wsp<int>(e, e->ws.slab_flag)) + 1 : nullptr;
  // the fallback only has to be correct; a small grid keeps the closed gate cheap
  const int chunks = gated ? 2 : (int)((e->ws.ldS / 4 + 256 * 8 - 1) / (256 * 8));
  if (is_3x(e))
    C2V_LAUNCH(e, (softmax_grad_kernel<true><<<dim3(chunks, B), 256, 0, st>>>(S, e->ws.ldS, Y, g.lse, g.target, g.inv_batch, g.row0,
                                                                             wsp<float>(e, e->ws.S_lo), gate, reset, count)));
  else
    C2V_LAUNCH(e, (softmax_grad_kernel<false><<<dim3(chunks, B), 256, 0, st>>>(S, e->ws.ldS, Y, g.lse, g.target, g.inv_batch, g.row0,
                                                                              nullptr, gate, reset, count)));
  if (gated) {
    float* vs = wsp<float>(e, e->ws.v_scaled);
    C2V_LAUNCH(e, (scale_rows_kernel<<<(unsigned)(((size_t)B * D + 255) / 256), 256, 0, st>>>(v, rscale, vs, D, (size_t)B * D)));
    slab->row_scale = rscale;
    *v_dy = vs;
  }
  return C2V_OK;
}

// exp_slab schedule (DESIGN.md section 4.9), up to the loss statistics: each row's true-class logit in fp32 (ws.true_logit,
// also copied to tl_out when given), the logits pass that writes U = exp(s - true logit) with (max U, sum U) partials, the
// caller's combine of those partials (it raises the range flag for rows that left the fp32 window), and the gated
// two-pass logits the device runs only for such rows.
template <class Combine>
int exp_slab_logits(c2v_engine* e, cudaStream_t st, const float* v, int B, const int32_t* target, int row0, float* tl_out,
                    Combine combine) {
  float* tl = wsp<float>(e, e->ws.true_logit);
  int* flag = wsp<int>(e, e->ws.slab_flag);
  if (!e->slab_flag_zeroed) {
    C2V_CUDA(e, cudaMemsetAsync(flag, 0, 64, st));
    e->slab_flag_zeroed = true;
  }
  int rc;
  if ((rc = end_target_lazy(e, st))) return rc;      // the true-class rows are read below: every target row must be current
  {
    PhaseTimer pt(e, PH_XENT, st);
    C2V_LAUNCH(e, (true_logit_kernel<<<(B + 7) / 8, 256, 0, st>>>(v, e->theta.tgt, target, row0, e->dims.target_vocab, e->dims.code_dim,
                                                                  B, tl, flag)));
    if (tl_out) C2V_CUDA(e, cudaMemcpyAsync(tl_out, tl, (size_t)B * 4, cudaMemcpyDeviceToDevice, st));
  }
  if ((rc = run_logits(e, st, v, B, LOGITS_EXP_SUM, LogitsArgs{tl}, true))) return rc;
  {
    PhaseTimer pt(e, PH_XENT, st);
    if ((rc = combine())) return rc;
  }
  return run_logits(e, st, v, B, LOGITS_STORE_LSE_GATED, LogitsArgs{nullptr, flag});
}

int train_step_impl(c2v_engine* e, cudaStream_t st, const int32_t* src, const int32_t* pth, const int32_t* tgt,
                    const float* mask, const int32_t* target, int B, float keep, uint64_t seed, uint64_t step,
                    const float* ext_mask, float* loss_out) {
  if (!e->has_grad) return fail(e, C2V_ERR_STATE, "gradients not bound (c2v_bind_grads)");
  if (!(keep > 0.f) || keep > 1.f) return fail(e, C2V_ERR_INVALID, "keep_prob must be in (0, 1]");
  const int Y = e->dims.target_vocab;
  const Dropout dp = make_dropout(e->dims, keep, seed, step, ext_mask);
  ContextSource cs = make_source(e, src, pth, tgt, B);
  float* H = wsp<float>(e, e->ws.H);
  float* alpha = wsp<float>(e, e->ws.alpha);
  float* v = wsp<float>(e, e->ws.v);
  float* dv = wsp<float>(e, e->ws.dv);
  float* S = wsp<float>(e, e->ws.S);
  float* loss_b = wsp<float>(e, e->ws.loss_b);
  float* lse = wsp<float>(e, e->ws.lse);
  float2* part = wsp<float2>(e, e->ws.lse_part);
  const int n_tiles = umma::lse_slots(Y);       // partial slots per row
  int rc;
  if ((rc = run_ctx_fwd(e, st, cs, dp, H, true))) return rc;
  if ((rc = launch_attn_fwd(e, st, H, mask, B, alpha, v))) return rc;
  const float invB = 1.0f / (float)B;
  const umma::SoftmaxGradArgs g{lse, target, 0, invB};
  const HeadSchedule hs = head_schedule(e, API_STEP, v);
  const float* v_dy = v;
  SlabDesc slab;
  if (hs == HEAD_RECOMPUTE) {
    // the slab is written ONCE, as dL/dlogits: pass 1 of the logits GEMM leaves only log-sum-exp partials, the true-class
    // logit comes from a B-row dot product, pass 2 repeats the product and its epilogue writes (softmax - onehot) / B
    if ((rc = run_logits(e, st, v, B, LOGITS_LSE_ONLY, {}, true))) return rc;
    float* tl = wsp<float>(e, e->ws.true_logit);
    {
      PhaseTimer pt(e, PH_XENT, st);
      C2V_LAUNCH(e, (true_logit_kernel<<<(B + 7) / 8, 256, 0, st>>>(v, e->theta.tgt, target, 0, Y, e->dims.code_dim, B, tl)));
      C2V_LAUNCH(e, (xent_combine_kernel<<<B, 256, 0, st>>>(part, n_tiles, S, e->ws.ldS, target, loss_b, lse, tl)));
      C2V_LAUNCH(e, (loss_reduce_kernel<<<1, 256, 0, st>>>(loss_b, B, invB, loss_out)));
    }
    if ((rc = run_logits(e, st, v, B, LOGITS_SOFTMAX_GRAD, LogitsArgs{nullptr, nullptr, g}))) return rc;
  } else if (hs == HEAD_EXP_SLAB) {
    // deferred normalisation: U = exp(s - true logit) from the logits epilogue, one patched element and one factor per row;
    // the gated kernels after the combine are the two-pass schedule, run by the device only when a row left the fp32 window
    float* tl = wsp<float>(e, e->ws.true_logit);
    float* rscale = wsp<float>(e, e->ws.rscale);
    int* flag = wsp<int>(e, e->ws.slab_flag);
    float* S_lo = is_3x(e) ? wsp<float>(e, e->ws.S_lo) : nullptr;
    rc = exp_slab_logits(e, st, v, B, target, 0, nullptr, [&]() -> int {
      C2V_LAUNCH(e, (expsum_combine_kernel<<<B, 256, 0, st>>>(part, n_tiles, S, S_lo, e->ws.ldS, Y, target, tl, tl, v, e->dims.code_dim,
                                                              invB, loss_b, lse, rscale, flag)));
      return C2V_OK;
    });
    if (rc) return rc;
    {
      PhaseTimer pt(e, PH_XENT, st);
      C2V_LAUNCH(e, (xent_combine_kernel<<<B, 256, 0, st>>>(part, n_tiles, S, e->ws.ldS, target, loss_b, lse, nullptr, flag, rscale,
                                                            reinterpret_cast<unsigned*>(flag) + 1)));
      if ((rc = slab_to_p(e, st, hs, v, B, g, &slab, &v_dy))) return rc;
      C2V_LAUNCH(e, (loss_reduce_kernel<<<1, 256, 0, st>>>(loss_b, B, invB, loss_out)));
    }
  } else {
    if ((rc = run_logits(e, st, v, B, hs == HEAD_SIMT ? LOGITS_STORE : LOGITS_STORE_LSE, {}, true))) return rc;
    PhaseTimer pt(e, PH_XENT, st);
    if (hs == HEAD_SIMT) {
      C2V_LAUNCH(e, (xent_kernel<<<B, kXentThreads, 0, st>>>(S, e->ws.ldS, target, Y, invB, loss_b, lse, 1)));
    } else {
      C2V_LAUNCH(e, (xent_combine_kernel<<<B, 256, 0, st>>>(part, n_tiles, S, e->ws.ldS, target, loss_b, lse)));
      if ((rc = slab_to_p(e, st, hs, v, B, g, &slab, &v_dy))) return rc;
    }
    C2V_LAUNCH(e, (loss_reduce_kernel<<<1, 256, 0, st>>>(loss_b, B, invB, loss_out)));
  }
  if ((rc = target_grad_gemms(e, st, v_dy, B, dv, slab))) return rc;
  return context_backward(e, st, cs, mask, B, dp, dv);
}

int sampled_train_step_impl(c2v_engine* e, cudaStream_t st, const int32_t* src, const int32_t* pth, const int32_t* tgt,
                             const float* mask, const int32_t* target, int B, const int32_t* sampled, int S,
                             const float* logq_true, const float* logq_samp, float keep, uint64_t seed, uint64_t step,
                             const float* ext_mask, float* loss_out) {
  if (!e->has_grad) return fail(e, C2V_ERR_STATE, "gradients not bound (c2v_bind_grads)");
  if (!(keep > 0.f) || keep > 1.f) return fail(e, C2V_ERR_INVALID, "keep_prob must be in (0, 1]");
  if (S < 1 || S > kMaxSampled) return fail(e, C2V_ERR_INVALID, "number of sampled classes must be in [1, 1024]");
  const int D = e->dims.code_dim;
  const Dropout dp = make_dropout(e->dims, keep, seed, step, ext_mask);
  ContextSource cs = make_source(e, src, pth, tgt, B);
  float* H = wsp<float>(e, e->ws.H);
  float* alpha = wsp<float>(e, e->ws.alpha);
  float* v = wsp<float>(e, e->ws.v);
  float* dv = wsp<float>(e, e->ws.dv);
  float* loss_b = wsp<float>(e, e->ws.loss_b);
  float* dl = wsp<float>(e, e->ws.dl);
  int rc;
  if ((rc = run_ctx_fwd(e, st, cs, dp, H, true))) return rc;
  if ((rc = launch_attn_fwd(e, st, H, mask, B, alpha, v))) return rc;
  const float invB = 1.0f / (float)B;
  if (e->lazy && e->has_adam && e->table_world == 1) {
    // TF1 applies sampled-softmax gradients as IndexedSlices: every row of the table still decays m, v and moves
    // (SURVEY A.3), exactly as for the embedding tables -- so the same deferred, bit-exact row replay applies, and
    // a step touches only the B + S rows it reads instead of streaming 24 B x 100 M parameters.
    PhaseTimer pt(e, PH_ADAM_CATCHUP, st);
    const c2v_dims& d = e->dims;
    int32_t* stamp = wsp<int32_t>(e, e->ws.stamp_tgt);
    int32_t* last = wsp<int32_t>(e, e->ws.last_tgt);
    if (!e->tgt_lazy) {          // the table joins the lazily updated set: every row is current as of adam_t_done
      C2V_CUDA(e, cudaMemsetAsync(e->grad.tgt, 0, (size_t)d.target_vocab * D * 4, st));
      C2V_LAUNCH(e, (fill_i32_kernel<<<256, 256, 0, st>>>(last, (size_t)d.target_vocab, (int32_t)e->adam_t_done)));
      C2V_CUDA(e, cudaMemsetAsync(stamp, 0, (size_t)d.target_vocab * 4, st));
      e->tgt_lazy = true;
    }
    e->mark_epoch++;
    C2V_LAUNCH(e, (mark_list_kernel<<<(B + 255) / 256, 256, 0, st>>>(target, B, stamp, e->mark_epoch)));
    C2V_LAUNCH(e, (mark_list_kernel<<<(S + 255) / 256, 256, 0, st>>>(sampled, S, stamp, e->mark_epoch)));
    if (e->adam_t_done > 0)
      C2V_ADAM_ROWS(e, ADAM_ROWS_CATCHUP, st,
                    e->theta.tgt, e->grad.tgt, e->am.tgt, e->av.tgt, d.target_vocab, d.code_dim, stamp, e->mark_epoch, last,
                    (int32_t)e->adam_t_done, wsp<float>(e, e->ws.lr_tab), e->hp_b1, e->hp_b2, e->hp_eps, rest_ok(e), pos_eps(e));
  }
  {
    PhaseTimer pt(e, PH_SAMPLED, st);
    const size_t smem = ((size_t)D + S + 1) * sizeof(float);
    C2V_LAUNCH(e, (sampled_softmax_fwd_kernel<<<B, kSampledThreads, smem, st>>>(v, e->theta.tgt, target, sampled, S, logq_true,
                                                                                 logq_samp, D, invB, loss_b, dl, dv)));
    C2V_LAUNCH(e, (loss_reduce_kernel<<<1, 256, 0, st>>>(loss_b, B, invB, loss_out)));
    // the target-table gradient is sparse here (B + S rows).  Lazy Adam: the rows were brought up to date (and
    // their gradient rows cleared) before the forward kernel read them; the update of this step is deferred
    // like an embedding row's.  Dense Adam: the bound buffer is dense, so it is cleared first.
    if (!e->tgt_lazy) C2V_CUDA(e, cudaMemsetAsync(e->grad.tgt, 0, (size_t)e->dims.target_vocab * D * 4, st));
    if (e->deterministic)     // one block per distinct row, terms in a fixed order, no atomics
      C2V_LAUNCH(e, (sampled_softmax_bwd_det_kernel<<<B + S, kSampledThreads, 0, st>>>(v, dl, target, sampled, B, S, D, e->grad.tgt)));
    else
      C2V_LAUNCH(e, (sampled_softmax_bwd_kernel<<<B + S * ((B + kSampledChunk - 1) / kSampledChunk), kSampledThreads, 0, st>>>(
          v, dl, target, sampled, B, S, D, e->grad.tgt)));
  }
  if (e->ev_tgt_ready) C2V_CUDA(e, cudaEventRecord(e->ev_tgt_ready, st));
  return context_backward(e, st, cs, mask, B, dp, dv);
}

int adam_impl(c2v_engine* e, cudaStream_t st, float lr, float b1, float b2, float eps, int64_t t) {
  if (!e->has_grad || !e->has_adam) return fail(e, C2V_ERR_STATE, "gradients / Adam state not bound");
  if (e->table_world > 1)
    return fail(e, C2V_ERR_STATE, "embedding tables are sharded: update each slice with c2v_adam_step_range");
  if (t < 1) return fail(e, C2V_ERR_INVALID, "Adam step count t must be >= 1");
  e->tgt_armed = false;                 // an unconsumed arming (fp32 path, sampled softmax) falls back to the dense update
  e->armed_t = 0;
  e->hint_src = e->hint_pth = e->hint_tgt = nullptr;      // a hint the step could not use is dropped
  bool skip_tgt = false;
  if (e->tgt_fused_t || e->early_t) {
    const int64_t done_t = e->tgt_fused_t ? e->tgt_fused_t : e->early_t;
    if (done_t != t || lr != e->tgt_lr || b1 != e->tgt_b1 || b2 != e->tgt_b2 || eps != e->tgt_eps)
      return fail(e, C2V_ERR_STATE, "part of this Adam step was already applied inside the train step (c2v_arm_target_adam) with a different step count / hyper-parameters");
    skip_tgt = e->tgt_fused_t != 0;
    e->tgt_fused_t = 0;
    e->early_t = 0;
  }
  const double lr_t_d = (double)lr * sqrt(1.0 - pow((double)b2, (double)t)) / (1.0 - pow((double)b1, (double)t));
  const float lr_t = (float)lr_t_d;
  const c2v_dims& d = e->dims;
  const size_t n[5] = {(size_t)d.token_vocab * d.embed_dim, (size_t)d.path_vocab * d.embed_dim,
                       (size_t)d.target_vocab * d.code_dim, (size_t)3 * d.embed_dim * d.code_dim, (size_t)d.code_dim};
  float* P[5] = {e->theta.tok, e->theta.path, e->theta.tgt, e->theta.W, e->theta.a};
  float* G[5] = {e->grad.tok, e->grad.path, e->grad.tgt, e->grad.W, e->grad.a};
  float* M[5] = {e->am.tok, e->am.path, e->am.tgt, e->am.W, e->am.a};
  float* V[5] = {e->av.tok, e->av.path, e->av.tgt, e->av.W, e->av.a};
  int first_dense = 0;
  if (e->lazy) {
    if (t != e->adam_t_done + 1) return fail(e, C2V_ERR_STATE, "lazy Adam needs consecutive step counts (t == previous t + 1)");
    if (e->hp_set && (lr != e->hp_lr || b1 != e->hp_b1 || b2 != e->hp_b2 || eps != e->hp_eps)) {
      int rcf = flush_rows(e, st);                  // pending steps must use the old hyper-parameters
      if (rcf) return rcf;
    }
    // the learning rates of pending steps live in a ring: no row may fall a whole ring behind (only possible
    // with the sweep switched off)
    if (t - e->full_flush_t >= kLrRing - 2) {
      int rcf = flush_rows(e, st);
      if (rcf) return rcf;
    }
    e->hp_lr = lr; e->hp_b1 = b1; e->hp_b2 = b2; e->hp_eps = eps; e->hp_set = true;
    float* lr_tab = wsp<float>(e, e->ws.lr_tab);
    // the embedding rows' step t is deferred: their gradient rows keep this step's scatter-add until the
    // rows are next referenced (prepare_rows), swept (sweep_rows) or flushed; only the learning rate of the
    // step is recorded
    C2V_LAUNCH(e, (set_float_kernel<<<1, 1, 0, st>>>(lr_tab + (t & kLrRingMask), lr_t)));
    e->lazy_grads_pending = false;
    first_dense = 2;
  }
  e->adam_t_done = t;
  e->tgt_t_valid = false;
  if (e->lazy) { int rcs = sweep_rows(e, st, t); if (rcs) return rcs; }
  for (int i = first_dense; i < 5; ++i) {
    if (i == 2 && (skip_tgt || e->tgt_lazy)) continue;     // lazy target rows: deferred like the embedding rows
    const size_t n4 = n[i] / 4;
    size_t blocks = (n4 + 255) / 256;
    if (blocks > (size_t)e->num_sms * 16) blocks = (size_t)e->num_sms * 16;
    if (blocks < 1) blocks = 1;
    const int zero = (i < 2) ? 1 : 0;   // embedding gradient tables are cleared for the next scatter-add
    PhaseTimer pt(e, PH_ADAM, st);
    C2V_LAUNCH(e, (adam_kernel<<<(unsigned)blocks, 256, 0, st>>>(P[i], G[i], M[i], V[i], n4, lr_t, b1, b2, eps, zero)));
  }
  e->emb_grads_clean = !e->lazy;     // lazy: the gradient tables hold deferred steps, cleared row by row as they are applied
  return C2V_OK;
}

}  // namespace

// failures of calls without an engine handle in other translation units (reader.cu): c2v_last_error(NULL) returns them
namespace c2v {
void set_global_error(const std::string& msg) { g_create_error = msg; }

// The top-k kernels of this file for the nearest-neighbour search (knn.cu), which cannot include kernels.cuh a second
// time.  Row r of `rows` keeps the best k of its L sorted candidate lists [L, k] at (idx, val) + r * L * k (k <= 16), or
// of slab row S + r * ldS (k <= 64), in tf.nn.top_k's order, into idx_out / val_out [rows, k].
cudaError_t knn_topk_merge(const int32_t* idx, const float* val, int L, int k, int rows, int32_t* idx_out, float* val_out,
                           cudaStream_t st) {
  const TopkMergeArgs ma{idx, val, L, (size_t)L * k, (size_t)k, k, 0, nullptr, nullptr, 1, rows, 0, idx_out, val_out};
  topk_merge_kernel<16><<<rows, kTopkThreads, 0, st>>>(ma);
  return cudaGetLastError();
}
cudaError_t launch_log_uniform_sampler(int32_t Y, double log_range, int32_t S, const int32_t* target, int32_t B,
                                       uint64_t seed, uint64_t step, uint32_t tag, unsigned long long* stamp,
                                       int32_t* sampled, float* logq_true, float* logq_sampled, int64_t* num_tries,
                                       int32_t* cap_hits, cudaStream_t st);     // sampler.cu
cudaError_t knn_topk_slab(const float* S, size_t ldS, int N, int k, int rows, int32_t* idx_out, float* val_out, cudaStream_t st) {
  if (k <= 16)
    topk_kernel<16><<<rows, kTopkThreads, 0, st>>>(S, ldS, N, k, 0, idx_out, val_out);
  else
    topk_iter_kernel<<<rows, kTopkThreads, 0, st>>>(S, ldS, N, k, 0, idx_out, val_out);
  return cudaGetLastError();
}
}

// ================================== C ABI =======================================================
extern "C" {

int c2v_abi_version(void) { return C2V_ABI_VERSION; }

const char* c2v_last_error(const c2v_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

size_t c2v_workspace_bytes(const c2v_dims* dims) {
  std::string why;
  if (!dims_ok(dims, &why)) { g_create_error = why; return 0; }
  return carve(*dims).total;
}

int c2v_create(const c2v_dims* dims, int device, c2v_engine** out) {
  if (!out) return fail(nullptr, C2V_ERR_INVALID, "out is NULL");
  *out = nullptr;
  std::string why;
  if (!dims_ok(dims, &why)) return fail(nullptr, C2V_ERR_INVALID, why);
  int ndev = 0;
  cudaError_t c = cudaGetDeviceCount(&ndev);
  if (c != cudaSuccess || ndev < 1)
    return fail(nullptr, C2V_ERR_CUDA, std::string("no CUDA device: ") + cudaGetErrorString(c));
  if (device < 0 || device >= ndev) return fail(nullptr, C2V_ERR_INVALID, "device ordinal out of range");
  cudaDeviceProp prop;
  c = cudaGetDeviceProperties(&prop, device);
  if (c != cudaSuccess) return fail(nullptr, C2V_ERR_CUDA, cudaGetErrorString(c));
  if (prop.major != 9 || prop.minor != 0)
    return fail(nullptr, C2V_ERR_UNSUPPORTED, "this library is built for sm_90a (H100) only");
  c2v_engine* e = new c2v_engine();
  e->dims = *dims;
  e->device = device;
  e->ws = carve(*dims);
  e->wbase = nullptr;
  e->wbytes = 0;
  e->has_theta = e->has_grad = e->has_adam = false;
  e->emb_grads_clean = false;
  e->math_mode = C2V_MATH_FP32;
  e->num_sms = prop.multiProcessorCount;
  cudaSetDevice(device);
  if (cudaStreamCreateWithFlags(&e->side, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_join, cudaEventDisableTiming) != cudaSuccess ||
      cudaStreamCreateWithFlags(&e->side2, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_fork2, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_join2, cudaEventDisableTiming) != cudaSuccess ||
      cudaStreamCreateWithFlags(&e->copy, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_h2d[0], cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_h2d[1], cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_used[0], cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_used[1], cudaEventDisableTiming) != cudaSuccess) {
    delete e;
    return fail(nullptr, C2V_ERR_CUDA, "could not create the engine's side stream / events");
  }
  e->deterministic = 0;
  e->launches = 0;
  *out = e;
  return C2V_OK;
}

void c2v_destroy(c2v_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  if (e->ev_fork) cudaEventDestroy(e->ev_fork);
  if (e->ev_join) cudaEventDestroy(e->ev_join);
  if (e->side) cudaStreamDestroy(e->side);
  if (e->ev_fork2) cudaEventDestroy(e->ev_fork2);
  if (e->ev_join2) cudaEventDestroy(e->ev_join2);
  if (e->side2) cudaStreamDestroy(e->side2);
  for (int i = 0; i < 2; ++i) {
    if (e->ev_h2d[i]) cudaEventDestroy(e->ev_h2d[i]);
    if (e->ev_used[i]) cudaEventDestroy(e->ev_used[i]);
  }
  if (e->copy) cudaStreamDestroy(e->copy);
  if (e->vstamp) cudaFree(e->vstamp);
  for (auto& L : e->phase) {
    for (auto& ev : L.pending) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
    for (auto& ev : L.free_list) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
  }
  delete e;
}

int c2v_bind_workspace(c2v_engine* e, void* dev_ptr, size_t bytes) {
  if (!e) return C2V_ERR_INVALID;
  if (!dev_ptr) return fail(e, C2V_ERR_INVALID, "workspace pointer is NULL");
  if (((uintptr_t)dev_ptr) % kAlign) return fail(e, C2V_ERR_INVALID, "workspace must be 256-byte aligned");
  if (bytes < e->ws.total) return fail(e, C2V_ERR_INVALID, "workspace smaller than c2v_workspace_bytes()");
  e->wbase = (char*)dev_ptr;
  e->wbytes = bytes;
  e->bkt_zeroed = false;
  e->slab_flag_zeroed = false;
  return C2V_OK;
}

int c2v_bind_params(c2v_engine* e, const c2v_tensors* t) {
  if (!e) return C2V_ERR_INVALID;
  if (!has_all(t)) return fail(e, C2V_ERR_INVALID, "all five parameter pointers must be non-NULL");
  e->theta = *t; e->has_theta = true;
  e->th_tok = ShardedTable{}; e->th_path = ShardedTable{};
  e->th_tok.base[0] = t->tok; e->th_path.base[0] = t->path;
  e->table_world = 1; e->grad_scale = 1.f;
  return C2V_OK;
}

int c2v_bind_grads(c2v_engine* e, const c2v_tensors* t) {
  if (!e) return C2V_ERR_INVALID;
  if (!has_all(t)) return fail(e, C2V_ERR_INVALID, "all five gradient pointers must be non-NULL");
  e->grad = *t; e->has_grad = true; e->emb_grads_clean = false;
  e->gr_tok = ShardedTable{}; e->gr_path = ShardedTable{};
  e->gr_tok.base[0] = t->tok; e->gr_path.base[0] = t->path;
  return C2V_OK;
}

int c2v_bind_adam_state(c2v_engine* e, const c2v_tensors* m, const c2v_tensors* v) {
  if (!e) return C2V_ERR_INVALID;
  if (!has_all(m) || !has_all(v)) return fail(e, C2V_ERR_INVALID, "all ten Adam slot pointers must be non-NULL");
  e->am = *m; e->av = *v; e->has_adam = true;
  return C2V_OK;
}

int c2v_set_option(c2v_engine* e, const char* key, int64_t value) {
  if (!e || !key) return C2V_ERR_INVALID;
  if (!strcmp(key, "math_mode")) {
    if (value != C2V_MATH_FP32 && value != C2V_MATH_TF32 && value != C2V_MATH_3XTF32)
      return fail(e, C2V_ERR_INVALID, "unknown math_mode");
    if (value != C2V_MATH_FP32 && !umma::get_encode_fn())
      return fail(e, C2V_ERR_UNSUPPORTED, "cuTensorMapEncodeTiled not available from the driver");
    e->math_mode = (int)value;
    e->tgt_t_valid = false;      // ws.tgtT holds the table (tf32) or its high parts (3xTF32)
    return C2V_OK;
  }
  if (!strcmp(key, "deterministic")) {
    if (value != 0 && value != 1) return fail(e, C2V_ERR_INVALID, "deterministic must be 0 or 1");
    if (value && e->table_world > 1 && !e->ordered_exchange)
      return fail(e, C2V_ERR_UNSUPPORTED, "deterministic: the embedding tables are row-sharded over more than one rank, and the "
                                          "cross-rank red.add scatter into them is order-free");
    if (value && (int64_t)e->dims.token_vocab + e->dims.path_vocab >= INT32_MAX)
      return fail(e, C2V_ERR_UNSUPPORTED, "deterministic: token_vocab + path_vocab must be below 2^31");
    e->deterministic = (int)value;
    return C2V_OK;
  }
  if (!strcmp(key, "ordered_exchange")) {
    if (value != 0 && value != 1) return fail(e, C2V_ERR_INVALID, "ordered_exchange must be 0 or 1");
    if (!value && e->deterministic && e->table_world > 1)
      return fail(e, C2V_ERR_UNSUPPORTED, "ordered_exchange: deterministic is set and the embedding tables are row-sharded over "
                                          "more than one rank; the other exchanges are order-free (set deterministic to 0 first)");
    if (value && !exchange_keys_fit(e->dims))
      return fail(e, C2V_ERR_UNSUPPORTED, "ordered_exchange: the padded rows of both tables over all ranks must be below 2^31");
    e->ordered_exchange = (int)value;
    return C2V_OK;
  }
  if (!strcmp(key, "profile")) { e->profile = value ? 1 : 0; return C2V_OK; }
  if (!strcmp(key, "dy_late")) {
    if (value < 0 || value > 2) return fail(e, C2V_ERR_INVALID, "dy_late must be 0, 1 or 2");
    e->dy_late = (int)value;
    return C2V_OK;
  }
  if (!strcmp(key, "fuse_target_adam")) { e->fuse_tgt = value ? 1 : 0; return C2V_OK; }
  if (!strcmp(key, "fuse_gather")) { e->fuse_gather = value ? 1 : 0; return C2V_OK; }
  if (!strcmp(key, "fuse_softmax_grad")) { e->fuse_sg = value ? 1 : 0; return C2V_OK; }
  if (!strcmp(key, "exp_slab")) { e->exp_slab = value ? 1 : 0; return C2V_OK; }
  if (!strcmp(key, "adam_epilogue_prefetch")) { e->adam_epi_prefetch = value ? 1 : 0; return C2V_OK; }
  if (!strcmp(key, "recompute_logits")) { e->recompute = value ? 1 : 0; return C2V_OK; }
  if (!strcmp(key, "sort_peer_access")) {
    if (value < 0 || value > 2) return fail(e, C2V_ERR_INVALID, "sort_peer_access must be 0 (never), 1 (auto) or 2 (always)");
    e->sort_peer = (int)value;
    return C2V_OK;
  }
  if (!strcmp(key, "adam_rest_shortcut")) { e->rest_shortcut = value ? 1 : 0; return C2V_OK; }
  if (!strcmp(key, "adam_sweep_period")) {
    if (value < 0 || value > kLrRing / 2) return fail(e, C2V_ERR_INVALID, "adam_sweep_period must be in [0, 32768]");
    e->sweep_period = (int)value;
    return C2V_OK;
  }
  if (!strcmp(key, "adam_rows_occupancy")) {
    if (value != 4 && value != 5) return fail(e, C2V_ERR_INVALID, "adam_rows_occupancy must be 4 or 5");
    e->adam_rows_occ = (int)value;
    return C2V_OK;
  }
  if (!strcmp(key, "cta_pair")) {
    if (value < 0 || value > 2) return fail(e, C2V_ERR_INVALID, "cta_pair must be 0 (never), 1 (always) or 2 (auto)");
    e->cta_pair = (int)value;
    return C2V_OK;
  }
  if (!strcmp(key, "grad_scale_inverse")) {               // scatter-add scale = 1 / value (1 = unscaled)
    if (value < 1) return fail(e, C2V_ERR_INVALID, "grad_scale_inverse must be >= 1");
    e->grad_scale = 1.0f / (float)value;
    return C2V_OK;
  }
  if (!strcmp(key, "lazy_adam")) {
    if (!e->wbase || !e->has_theta || !e->has_grad || !e->has_adam)
      return fail(e, C2V_ERR_STATE, "bind workspace, parameters, gradients and Adam state before lazy_adam");
    if (value && e->table_world > 1) return fail(e, C2V_ERR_STATE, "lazy_adam is for replicated (single-GPU) tables");
    C2V_CUDA(e, cudaSetDevice(e->device));
    if (!value && e->lazy) {                              // bring every row up to date, then go dense
      int rc = flush_rows(e, 0);
      if (rc) return rc;
      C2V_CUDA(e, cudaStreamSynchronize(0));
      e->emb_grads_clean = !e->lazy_grads_pending;        // every applied gradient row was cleared on the way
      e->lazy_grads_pending = false;
      e->tgt_lazy = false;
    }
    if (value && !e->lazy) {                              // all rows are current as of adam_t_done
      const c2v_dims& d = e->dims;
      if (!e->emb_grads_clean) {                          // deferred steps read the gradient rows: they must start from zero
        C2V_CUDA(e, cudaMemset(e->grad.tok, 0, (size_t)d.token_vocab * d.embed_dim * 4));
        C2V_CUDA(e, cudaMemset(e->grad.path, 0, (size_t)d.path_vocab * d.embed_dim * 4));
      }
      e->lazy_grads_pending = false;
      C2V_LAUNCH(e, (fill_i32_kernel<<<256, 256>>>(wsp<int32_t>(e, e->ws.last_tok), (size_t)d.token_vocab, (int32_t)e->adam_t_done)));
      C2V_LAUNCH(e, (fill_i32_kernel<<<256, 256>>>(wsp<int32_t>(e, e->ws.last_path), (size_t)d.path_vocab, (int32_t)e->adam_t_done)));
      C2V_CUDA(e, cudaMemset(wsp<int32_t>(e, e->ws.stamp_tok), 0, (size_t)d.token_vocab * 4));
      C2V_CUDA(e, cudaMemset(wsp<int32_t>(e, e->ws.stamp_path), 0, (size_t)d.path_vocab * 4));
      e->mark_epoch = 0;
      e->full_flush_t = e->adam_t_done;
      e->tgt_lazy = false;
      C2V_CUDA(e, cudaDeviceSynchronize());
    }
    e->lazy = value ? 1 : 0;
    return C2V_OK;
  }
  if (!strcmp(key, "target_adam_fused_step")) {           // callers that run c2v_adam_step_range themselves acknowledge with 0
    if (value) return fail(e, C2V_ERR_INVALID, "target_adam_fused_step can only be cleared (0)");
    e->tgt_fused_t = 0;
    return C2V_OK;
  }
  if (!strcmp(key, "adam_step_count")) {                  // optimizer reset / checkpoint restore
    C2V_CUDA(e, cudaSetDevice(e->device));
    if (e->lazy) {
      int rc = flush_rows(e, 0);
      if (rc) return rc;
      const c2v_dims& d = e->dims;
      C2V_LAUNCH(e, (fill_i32_kernel<<<256, 256>>>(wsp<int32_t>(e, e->ws.last_tok), (size_t)d.token_vocab, (int32_t)value)));
      C2V_LAUNCH(e, (fill_i32_kernel<<<256, 256>>>(wsp<int32_t>(e, e->ws.last_path), (size_t)d.path_vocab, (int32_t)value)));
      C2V_CUDA(e, cudaDeviceSynchronize());
      e->tgt_lazy = false;                                // flush_rows brought the target rows up to date as well
      e->full_flush_t = value;
    }
    e->adam_t_done = value;
    e->hp_set = false;
    return C2V_OK;
  }
  return fail(e, C2V_ERR_INVALID, std::string("unknown option: ") + key);
}

int c2v_get_option(const c2v_engine* e, const char* key, int64_t* value) {
  if (!e || !key || !value) return C2V_ERR_INVALID;
  if (!strcmp(key, "math_mode")) { *value = e->math_mode; return C2V_OK; }
  if (!strcmp(key, "deterministic")) { *value = e->deterministic; return C2V_OK; }
  if (!strcmp(key, "ordered_exchange")) { *value = e->ordered_exchange; return C2V_OK; }
  if (!strcmp(key, "ordered_exchange_rows")) {    // (row, sum) records this rank pushed in its last step, over all owners (synchronises)
    *value = 0;
    if (e->wbase && e->exchange_pushed) {
      int32_t n = 0;
      if (cudaDeviceSynchronize() != cudaSuccess ||
          cudaMemcpy(&n, e->wbase + e->ws.det_starts + (size_t)2 * e->table_world * 4, 4, cudaMemcpyDeviceToHost) != cudaSuccess)
        return C2V_ERR_CUDA;
      *value = n;
    }
    return C2V_OK;
  }
  if (!strcmp(key, "profile")) { *value = e->profile; return C2V_OK; }
  if (!strcmp(key, "lazy_adam")) { *value = e->lazy; return C2V_OK; }
  if (!strcmp(key, "adam_sweep_period")) { *value = e->sweep_period; return C2V_OK; }
  if (!strcmp(key, "adam_rest_shortcut")) { *value = e->rest_shortcut; return C2V_OK; }
  if (!strcmp(key, "cta_pair")) { *value = e->cta_pair; return C2V_OK; }
  if (!strcmp(key, "dy_late")) { *value = e->dy_late; return C2V_OK; }
  if (!strcmp(key, "fuse_target_adam")) { *value = e->fuse_tgt; return C2V_OK; }
  if (!strcmp(key, "fuse_gather")) { *value = e->fuse_gather; return C2V_OK; }
  if (!strcmp(key, "fuse_softmax_grad")) { *value = e->fuse_sg; return C2V_OK; }
  if (!strcmp(key, "exp_slab")) { *value = e->exp_slab; return C2V_OK; }
  if (!strcmp(key, "adam_epilogue_prefetch")) { *value = e->adam_epi_prefetch; return C2V_OK; }
  if (!strcmp(key, "exp_slab_fallbacks")) {       // steps so far that left the fp32 window and ran the two-pass schedule (synchronises)
    *value = 0;
    if (e->wbase && e->slab_flag_zeroed) {
      unsigned n = 0;
      if (cudaDeviceSynchronize() != cudaSuccess ||
          cudaMemcpy(&n, e->wbase + e->ws.slab_flag + 4, 4, cudaMemcpyDeviceToHost) != cudaSuccess)
        return C2V_ERR_CUDA;
      *value = n;
    }
    return C2V_OK;
  }
  if (!strcmp(key, "sampler_cap_hits")) {         // sampler calls (either entry point) that reached the draw cap (synchronises)
    *value = 0;
    if (e->wbase && e->cap_hits_zeroed) {
      int32_t n = 0;
      if (cudaDeviceSynchronize() != cudaSuccess ||
          cudaMemcpy(&n, e->wbase + e->ws.samp_status, 4, cudaMemcpyDeviceToHost) != cudaSuccess)
        return C2V_ERR_CUDA;
      *value = n;
    }
    return C2V_OK;
  }
  if (!strcmp(key, "recompute_logits")) { *value = e->recompute; return C2V_OK; }
  if (!strcmp(key, "sort_peer_access")) { *value = e->sort_peer; return C2V_OK; }
  if (!strcmp(key, "adam_step_count")) { *value = e->adam_t_done; return C2V_OK; }
  if (!strcmp(key, "target_adam_fused_step")) { *value = e->tgt_fused_t; return C2V_OK; }
  if (!strcmp(key, "early_catchup_count")) { *value = e->early_count; return C2V_OK; }
  return C2V_ERR_INVALID;
}

int c2v_forward(c2v_engine* e, const int32_t* src, const int32_t* path, const int32_t* tgt, const float* mask,
                int32_t B, float* code_vec, float* attn, void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!src || !path || !tgt || !mask || !code_vec) return fail(e, C2V_ERR_INVALID, "NULL argument");
  C2V_CUDA(e, cudaSetDevice(e->device));
  const Dropout dp = make_dropout(e->dims, 1.0f, 0, 0, nullptr);
  return forward_impl(e, (cudaStream_t)stream, src, path, tgt, mask, B, dp, code_vec, attn);
}

int c2v_topk(c2v_engine* e, const float* code_vec, int32_t B, int32_t* idx, float* val, int32_t normalize,
             void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!code_vec || !idx || !val) return fail(e, C2V_ERR_INVALID, "NULL argument");
  C2V_CUDA(e, cudaSetDevice(e->device));
  return topk_impl(e, (cudaStream_t)stream, code_vec, B, idx, val, normalize);
}

int c2v_topk_partial(c2v_engine* e, const float* code_all, int32_t Bt, int32_t row_offset, int32_t k, int32_t* idx, float* val,
                     float* row_max, float* row_sum, void* stream) {
  int rc = check_batch(e, Bt);
  if (rc) return rc;
  if (!code_all || !idx || !val) return fail(e, C2V_ERR_INVALID, "NULL argument");
  if ((row_max == nullptr) != (row_sum == nullptr)) return fail(e, C2V_ERR_INVALID, "row_max and row_sum: both or neither");
  if (k < 1 || k > e->dims.top_k) return fail(e, C2V_ERR_INVALID, "k must be in [1, top_k]");
  if (row_offset < 0) return fail(e, C2V_ERR_INVALID, "row_offset must be >= 0");
  C2V_CUDA(e, cudaSetDevice(e->device));
  return topk_partial_impl(e, (cudaStream_t)stream, code_all, Bt, row_offset, k, idx, val, row_max, row_sum);
}

int c2v_topk_merge(c2v_engine* e, const int32_t* idx, const float* val, const float* maxes, const float* sums, int32_t world,
                   int32_t Bt, int32_t k, int32_t row0, int32_t rows, int32_t normalize, int32_t* idx_out, float* val_out,
                   void* stream) {
  if (!e) return C2V_ERR_INVALID;
  if (!idx || !val || !idx_out || !val_out) return fail(e, C2V_ERR_INVALID, "NULL argument");
  if (normalize < 0 || normalize > 2) return fail(e, C2V_ERR_INVALID, "normalize must be 0 (logits), 1 (softmax over k) or 2 (full softmax)");
  if (normalize == 2 && (!maxes || !sums)) return fail(e, C2V_ERR_INVALID, "normalize 2 needs maxes and sums");
  if (world < 1 || Bt < 1 || k < 1 || k > e->dims.top_k) return fail(e, C2V_ERR_INVALID, "bad size");
  if (rows < 1 || row0 < 0 || row0 > Bt - rows) return fail(e, C2V_ERR_INVALID, "rows [row0, row0 + rows) must lie in [0, Bt)");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  PhaseTimer pt(e, PH_TOPK, st);
  // list r of row b: idx[r, b, :]
  const TopkMergeArgs ma{idx, val, world, (size_t)k, (size_t)Bt * k, k, normalize, maxes, sums, world, Bt, row0, idx_out, val_out};
  if (k <= 16)
    C2V_LAUNCH(e, (topk_merge_kernel<16><<<rows, kTopkThreads, 0, st>>>(ma)));
  else
    C2V_LAUNCH(e, (topk_merge_iter_kernel<<<rows, kTopkThreads, 0, st>>>(ma)));
  return C2V_OK;
}

int c2v_loss(c2v_engine* e, const float* code_vec, const int32_t* target, int32_t B, float* loss_out, void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!code_vec || !target || !loss_out) return fail(e, C2V_ERR_INVALID, "NULL argument");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  float* S = wsp<float>(e, e->ws.S);
  const float invB = 1.0f / (float)B;
  const int Y = e->dims.target_vocab;
  const bool fused = head_schedule(e, API_LOSS, code_vec) == HEAD_TWO_PASS;
  if ((rc = run_logits(e, st, code_vec, B, fused ? LOGITS_STORE_LSE : LOGITS_STORE))) return rc;
  {
    PhaseTimer pt(e, PH_XENT, st);
    if (fused)      // the logits epilogue already folded each tile into (max, sum exp) partials
      C2V_LAUNCH(e, (xent_combine_kernel<<<B, 256, 0, st>>>(wsp<float2>(e, e->ws.lse_part), umma::lse_slots(Y), S, e->ws.ldS, target,
                                                            wsp<float>(e, e->ws.loss_b), wsp<float>(e, e->ws.lse))));
    else
      C2V_LAUNCH(e, (xent_kernel<<<B, kXentThreads, 0, st>>>(S, e->ws.ldS, target, Y, invB, wsp<float>(e, e->ws.loss_b),
                                                              wsp<float>(e, e->ws.lse), 0)));
    C2V_LAUNCH(e, (loss_reduce_kernel<<<1, 256, 0, st>>>(wsp<float>(e, e->ws.loss_b), B, invB, loss_out)));
  }
  return C2V_OK;
}

int c2v_name_scores(c2v_engine* e, const float* code_vec, const int32_t* target, int32_t B, int32_t* rank, float* logp,
                    int32_t* top1, float* top1_logp, void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!code_vec || !target || !rank || !logp || !top1 || !top1_logp) return fail(e, C2V_ERR_INVALID, "NULL argument");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = run_logits(e, st, code_vec, B, LOGITS_STORE))) return rc;       // the slab topk_impl scans, bit for bit
  PhaseTimer pt(e, PH_NAME_RANK, st);
  C2V_LAUNCH(e, (name_rank_kernel<<<B, kNameRankThreads, 0, st>>>(wsp<float>(e, e->ws.S), e->ws.ldS, e->dims.target_vocab,
                                                                     target, rank, logp, top1, top1_logp)));
  return C2V_OK;
}

int c2v_train_step(c2v_engine* e, const int32_t* src, const int32_t* path, const int32_t* tgt, const float* mask,
                   const int32_t* target, int32_t B, float keep_prob, uint64_t seed, uint64_t step,
                   const float* dropout_mask, float* loss_out, void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!src || !path || !tgt || !mask || !target || !loss_out) return fail(e, C2V_ERR_INVALID, "NULL argument");
  C2V_CUDA(e, cudaSetDevice(e->device));
  return train_step_impl(e, (cudaStream_t)stream, src, path, tgt, mask, target, B, keep_prob, seed, step,
                         dropout_mask, loss_out);
}

int c2v_sampled_train_step(c2v_engine* e, const int32_t* src, const int32_t* path, const int32_t* tgt, const float* mask,
                           const int32_t* target, int32_t B, const int32_t* sampled, int32_t S, const float* logq_true,
                           const float* logq_sampled, float keep_prob, uint64_t seed, uint64_t step,
                           const float* dropout_mask, float* loss_out, void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!src || !path || !tgt || !mask || !target || !sampled || !logq_true || !logq_sampled || !loss_out)
    return fail(e, C2V_ERR_INVALID, "NULL argument");
  C2V_CUDA(e, cudaSetDevice(e->device));
  return sampled_train_step_impl(e, (cudaStream_t)stream, src, path, tgt, mask, target, B, sampled, S, logq_true,
                                 logq_sampled, keep_prob, seed, step, dropout_mask, loss_out);
}

int c2v_sample_log_uniform(c2v_engine* e, int32_t S, const int32_t* target, int32_t B, uint64_t seed, uint64_t step,
                           int32_t* sampled, float* logq_true, float* logq_sampled, int64_t* num_tries, void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!target || !sampled || !logq_true || !logq_sampled) return fail(e, C2V_ERR_INVALID, "NULL argument");
  const int32_t Y = e->dims.target_vocab;
  if (S < 1 || S > kMaxSampled || S > Y / 2)
    return fail(e, C2V_ERR_INVALID, "number of sampled classes must be in [1, min(1024, target_vocab / 2)]");
  if (e->table_world > 1)
    return fail(e, C2V_ERR_UNSUPPORTED, "c2v_sample_log_uniform is single-GPU: the tables are row-sharded over several ranks");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* stamp = wsp<unsigned long long>(e, e->ws.samp_stamp);
  int32_t* cap_hits = wsp<int32_t>(e, e->ws.samp_status);
  // a call's stamps are (tag << 32 | draw index) with tags counting down, so every earlier call's stamp is larger and the
  // table never needs clearing -- except once at the start and after the 2^32 - 2 tags are used up
  if (e->sample_tag <= 1) {
    C2V_CUDA(e, cudaMemsetAsync(stamp, 0xFF, (size_t)Y * 8, st));
    e->sample_tag = 0xFFFFFFFFu;
  }
  if (!e->cap_hits_zeroed) {
    C2V_CUDA(e, cudaMemsetAsync(cap_hits, 0, 4, st));
    e->cap_hits_zeroed = true;
  }
  e->sample_tag--;
  PhaseTimer pt(e, PH_SAMPLER, st);
  C2V_LAUNCH(e, C2V_CUDA(e, launch_log_uniform_sampler(Y, log1p((double)Y), S, target, B, seed, step, e->sample_tag, stamp,
                                                       sampled, logq_true, logq_sampled, num_tries, cap_hits, st)));
  return C2V_OK;
}

int c2v_sample_log_uniform_vocab(c2v_engine* e, int32_t S, int32_t Y, const int32_t* target, int32_t B, uint64_t seed,
                                 uint64_t step, int32_t* sampled, float* logq_true, float* logq_sampled, int64_t* num_tries,
                                 void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!target || !sampled || !logq_true || !logq_sampled) return fail(e, C2V_ERR_INVALID, "NULL argument");
  if (Y < 2) return fail(e, C2V_ERR_INVALID, "the target vocabulary needs at least 2 classes");
  if (S < 1 || S > kMaxSampled || S > Y / 2)
    return fail(e, C2V_ERR_INVALID, "number of sampled classes must be in [1, min(1024, Y / 2)]");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  if (Y > e->vstamp_Y) {            // the first call (or a larger vocabulary): the stamp table is this call's own allocation
    if (e->vstamp) {
      C2V_CUDA(e, cudaStreamSynchronize(st));
      C2V_CUDA(e, cudaFree(e->vstamp));
      e->vstamp = nullptr;
      e->vstamp_Y = 0;
    }
    C2V_CUDA(e, cudaMalloc((void**)&e->vstamp, (size_t)Y * 8));
    e->vstamp_Y = Y;
    e->vsample_tag = 0;
  }
  int32_t* cap_hits = wsp<int32_t>(e, e->ws.samp_status);
  if (e->vsample_tag <= 1) {        // tags count down as in c2v_sample_log_uniform
    C2V_CUDA(e, cudaMemsetAsync(e->vstamp, 0xFF, (size_t)e->vstamp_Y * 8, st));
    e->vsample_tag = 0xFFFFFFFFu;
  }
  if (!e->cap_hits_zeroed) {
    C2V_CUDA(e, cudaMemsetAsync(cap_hits, 0, 4, st));
    e->cap_hits_zeroed = true;
  }
  e->vsample_tag--;
  PhaseTimer pt(e, PH_SAMPLER, st);
  C2V_LAUNCH(e, C2V_CUDA(e, launch_log_uniform_sampler(Y, log1p((double)Y), S, target, B, seed, step, e->vsample_tag, e->vstamp,
                                                       sampled, logq_true, logq_sampled, num_tries, cap_hits, st)));
  return C2V_OK;
}

int c2v_arm_target_adam(c2v_engine* e, float lr, float beta1, float beta2, float eps, int64_t t) {
  if (!e) return C2V_ERR_INVALID;
  if (!e->has_theta || !e->has_adam) return fail(e, C2V_ERR_STATE, "parameters / Adam state not bound");
  if (t < 1) return fail(e, C2V_ERR_INVALID, "Adam step count t must be >= 1");
  if (e->tgt_fused_t)
    return fail(e, C2V_ERR_STATE, "a fused target update is still unacknowledged: call c2v_adam_step (or clear target_adam_fused_step)");
  if (e->early_t) return fail(e, C2V_ERR_STATE, "the previous armed step is still unacknowledged: call c2v_adam_step");
  e->tgt_lr = lr; e->tgt_b1 = beta1; e->tgt_b2 = beta2; e->tgt_eps = eps; e->tgt_t = t;
  e->tgt_armed = true;
  e->armed_t = t;
  return C2V_OK;
}

int c2v_hint_next_batch(c2v_engine* e, const int32_t* src, const int32_t* path, const int32_t* tgt, int32_t B) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!src || !path || !tgt) return fail(e, C2V_ERR_INVALID, "NULL argument");
  e->hint_src = src; e->hint_pth = path; e->hint_tgt = tgt; e->hint_B = B;
  return C2V_OK;
}

int c2v_hint_next_batch_host(c2v_engine* e, const int32_t* h_src, const int32_t* h_path, const int32_t* h_tgt, int32_t B,
                             void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!h_src || !h_path || !h_tgt) return fail(e, C2V_ERR_INVALID, "NULL argument");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t nb = (size_t)B * e->dims.max_contexts * 4;
  int32_t* src = wsp<int32_t>(e, e->ws.nx_src);
  int32_t* pth = wsp<int32_t>(e, e->ws.nx_pth);
  int32_t* tgt = wsp<int32_t>(e, e->ws.nx_tgt);
  C2V_CUDA(e, cudaMemcpyAsync(src, h_src, nb, cudaMemcpyHostToDevice, st));
  C2V_CUDA(e, cudaMemcpyAsync(pth, h_path, nb, cudaMemcpyHostToDevice, st));
  C2V_CUDA(e, cudaMemcpyAsync(tgt, h_tgt, nb, cudaMemcpyHostToDevice, st));
  return c2v_hint_next_batch(e, src, pth, tgt, B);
}

int c2v_adam_step(c2v_engine* e, float lr, float beta1, float beta2, float eps, int64_t t, void* stream) {
  if (!e) return C2V_ERR_INVALID;
  if (!e->has_theta) return fail(e, C2V_ERR_STATE, "parameters not bound");
  C2V_CUDA(e, cudaSetDevice(e->device));
  return adam_impl(e, (cudaStream_t)stream, lr, beta1, beta2, eps, t);
}

int c2v_bind_table_shards(c2v_engine* e, const c2v_table_shards* params, const c2v_table_shards* grads, float grad_scale) {
  if (!e) return C2V_ERR_INVALID;
  if (!params) return fail(e, C2V_ERR_INVALID, "params shards are NULL");
  if (!e->has_theta) return fail(e, C2V_ERR_STATE, "bind the replicated tensors first (c2v_bind_params)");
  const int w = params->world;
  if (!(w == 1 || w == 2 || w == 4 || w == 8)) return fail(e, C2V_ERR_INVALID, "world must be 1, 2, 4 or 8");
  if (grads && grads->world != w) return fail(e, C2V_ERR_INVALID, "params / grads world mismatch");
  if (e->deterministic && w > 1 && !e->ordered_exchange)
    return fail(e, C2V_ERR_UNSUPPORTED, "deterministic is set: row-sharded tables over more than one rank take order-free "
                                        "cross-rank red.adds (set deterministic to 0 first)");
  int shift = 0;
  while ((1 << shift) < w) ++shift;
  auto fill = [&](ShardedTable& t, float* const* ptrs) -> bool {
    t = ShardedTable{};
    t.shift = shift; t.mask = w - 1;
    for (int i = 0; i < w; ++i) { if (!ptrs[i]) return false; t.base[i] = ptrs[i]; }
    return true;
  };
  if (!fill(e->th_tok, params->tok) || !fill(e->th_path, params->path)) return fail(e, C2V_ERR_INVALID, "NULL shard pointer");
  if (grads) {
    if (!fill(e->gr_tok, grads->tok) || !fill(e->gr_path, grads->path)) return fail(e, C2V_ERR_INVALID, "NULL shard pointer");
  }
  e->table_world = w;
  e->grad_scale = grad_scale;
  return C2V_OK;
}

size_t c2v_scatter_inbox_bytes(const c2v_dims* dims, int32_t world) {
  std::string why;
  if (!dims_ok(dims, &why) || world < 1 || world > kMaxShards) { g_create_error = why.empty() ? "bad world" : why; return 0; }
  const size_t cap = (size_t)3 * dims->max_batch * dims->max_contexts;
  return inbox_val_offset(world, cap) + (size_t)world * cap * dims->embed_dim * 4;
}

int c2v_bind_scatter_inbox(c2v_engine* e, void* const* inbox, int32_t world, int32_t rank) {
  if (!e) return C2V_ERR_INVALID;
  if (!inbox) { e->inbox = InboxSet{}; return C2V_OK; }           // unbind: back to remote red.add
  if (world != e->table_world || world < 2) return fail(e, C2V_ERR_STATE, "bind the table shards first (same world)");
  if (rank < 0 || rank >= world) return fail(e, C2V_ERR_INVALID, "rank out of range");
  InboxSet s{};
  for (int i = 0; i < world; ++i) {
    if (!inbox[i]) return fail(e, C2V_ERR_INVALID, "NULL inbox pointer");
    s.base[i] = (char*)inbox[i];
  }
  s.cap = (size_t)3 * e->dims.max_batch * e->dims.max_contexts;
  s.world = world; s.rank = rank;
  e->inbox = s;
  return C2V_OK;
}

int c2v_apply_scatter_inbox(c2v_engine* e, void* stream) {
  if (!e) return C2V_ERR_INVALID;
  if (e->inbox.world < 2) return fail(e, C2V_ERR_STATE, "no scatter inbox bound (c2v_bind_scatter_inbox)");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  PhaseTimer pt(e, PH_INBOX_APPLY, st);
  float* g_tok = e->gr_tok.base[e->inbox.rank];
  float* g_path = e->gr_path.base[e->inbox.rank];
  if (ordered_route(e))        // the senders' sorted row sums, added per row in sender order and stored
    C2V_LAUNCH(e, (inbox_fold_ordered_kernel<<<e->num_sms * 8, 256, 0, st>>>(e->inbox, e->dims.embed_dim, g_tok, g_path)));
  else
    C2V_LAUNCH(e, (inbox_apply_kernel<<<e->num_sms * 8, 256, 0, st>>>(e->inbox, e->dims.embed_dim, g_tok, g_path)));
  // the fold consumes the rows: a step that pushes nothing (the fp32 scatter red.adds straight into the shards) leaves
  // zero counts, so the next fold cannot add the previous step's rows a second time
  C2V_CUDA(e, cudaMemsetAsync(e->inbox.base[e->inbox.rank], 0, (size_t)e->inbox.world * 2 * 4, st));
  return C2V_OK;
}

int c2v_ipc_alloc(int device, size_t bytes, void** dev_ptr, unsigned char* handle64) {
  if (!dev_ptr || !handle64 || bytes == 0) return fail(nullptr, C2V_ERR_INVALID, "bad argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  C2V_CUDA((c2v_engine*)nullptr, cudaSetDevice(device));
  C2V_CUDA((c2v_engine*)nullptr, cudaMalloc(dev_ptr, bytes));
  C2V_CUDA((c2v_engine*)nullptr, cudaMemset(*dev_ptr, 0, bytes));
  cudaIpcMemHandle_t h;
  C2V_CUDA((c2v_engine*)nullptr, cudaIpcGetMemHandle(&h, *dev_ptr));
  memcpy(handle64, &h, 64);
  return C2V_OK;
}

int c2v_ipc_open(int device, const unsigned char* handle64, void** dev_ptr) {
  if (!dev_ptr || !handle64) return fail(nullptr, C2V_ERR_INVALID, "bad argument");
  C2V_CUDA((c2v_engine*)nullptr, cudaSetDevice(device));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  C2V_CUDA((c2v_engine*)nullptr, cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return C2V_OK;
}

int c2v_ipc_close(int device, void* dev_ptr) {
  C2V_CUDA((c2v_engine*)nullptr, cudaSetDevice(device));
  C2V_CUDA((c2v_engine*)nullptr, cudaIpcCloseMemHandle(dev_ptr));
  return C2V_OK;
}

int c2v_ipc_free(int device, void* dev_ptr) {
  C2V_CUDA((c2v_engine*)nullptr, cudaSetDevice(device));
  C2V_CUDA((c2v_engine*)nullptr, cudaFree(dev_ptr));
  return C2V_OK;
}

// ---- phase-split training step: the fully sharded schedule (target table row-sharded too) ------------
int c2v_context_forward(c2v_engine* e, const int32_t* src, const int32_t* path, const int32_t* tgt, const float* mask,
                        int32_t B, float keep_prob, uint64_t seed, uint64_t step, const float* dropout_mask,
                        float* code_vec, void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!src || !path || !tgt || !mask || !code_vec) return fail(e, C2V_ERR_INVALID, "NULL argument");
  if (!(keep_prob > 0.f) || keep_prob > 1.f) return fail(e, C2V_ERR_INVALID, "keep_prob must be in (0, 1]");
  C2V_CUDA(e, cudaSetDevice(e->device));
  const Dropout dp = make_dropout(e->dims, keep_prob, seed, step, dropout_mask);
  return forward_impl(e, (cudaStream_t)stream, src, path, tgt, mask, B, dp, code_vec, wsp<float>(e, e->ws.alpha), true);
}

int c2v_target_forward(c2v_engine* e, const float* code_all, int32_t Bt, const int32_t* target, int32_t row_offset,
                       float* row_max, float* row_sum, float* true_logit, void* stream) {
  int rc = check_batch(e, Bt);
  if (rc) return rc;
  if (!code_all || !target || !row_max || !row_sum || !true_logit) return fail(e, C2V_ERR_INVALID, "NULL argument");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  float* S = wsp<float>(e, e->ws.S);
  const int Y = e->dims.target_vocab;
  const int n_tiles = umma::lse_slots(Y);
  float2* part = wsp<float2>(e, e->ws.lse_part);
  const HeadSchedule hs = head_schedule(e, API_TARGET_FORWARD, code_all);
  e->split_fwd = hs;
  if (hs == HEAD_EXP_SLAB) {
    // deferred normalisation over a row-sharded table: (c_b, sum U) stand in for (row max, sum exp) in the cross-rank combine;
    // a row that left the fp32 window has the statistics that go to the other ranks redone the classic way
    float* tl = wsp<float>(e, e->ws.true_logit);
    int* flag = wsp<int>(e, e->ws.slab_flag);
    rc = exp_slab_logits(e, st, code_all, Bt, target, row_offset, true_logit, [&]() -> int {
      C2V_LAUNCH(e, (expsum_rows_kernel<<<Bt, 256, 0, st>>>(part, n_tiles, tl, row_max, row_sum, flag)));
      return C2V_OK;
    });
    if (rc) return rc;
    PhaseTimer pt(e, PH_XENT, st);
    C2V_LAUNCH(e, (row_maxsum_kernel<<<Bt, 256, 0, st>>>(part, n_tiles, S, e->ws.ldS, Y, target, row_offset, row_max, row_sum, true_logit,
                                                         1, flag)));
    return C2V_OK;
  }
  const bool fused = hs == HEAD_TWO_PASS;
  if ((rc = run_logits(e, st, code_all, Bt, fused ? LOGITS_STORE_LSE : LOGITS_STORE, {}, true))) return rc;
  PhaseTimer pt(e, PH_XENT, st);
  C2V_LAUNCH(e, (row_maxsum_kernel<<<Bt, 256, 0, st>>>(fused ? part : nullptr, n_tiles, S, e->ws.ldS, Y, target, row_offset, row_max,
                                                       row_sum, true_logit)));
  return C2V_OK;
}

int c2v_lse_combine(c2v_engine* e, const float* maxes, const float* sums, int32_t world, int32_t Bt, const float* true_logit,
                    float inv_batch, float* lse_out, float* loss_out, void* stream) {
  if (!e || !maxes || !sums || !true_logit || !lse_out || !loss_out) return C2V_ERR_INVALID;
  if (Bt < 1 || Bt > e->dims.max_batch || world < 1) return fail(e, C2V_ERR_INVALID, "bad size");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  float* loss_b = wsp<float>(e, e->ws.loss_b);
  C2V_LAUNCH(e, (lse_combine_kernel<<<(Bt + 255) / 256, 256, 0, st>>>(maxes, sums, world, Bt, true_logit, lse_out, loss_b)));
  C2V_LAUNCH(e, (loss_reduce_kernel<<<1, 256, 0, st>>>(loss_b, Bt, inv_batch, loss_out)));
  return C2V_OK;
}

int c2v_target_backward(c2v_engine* e, const float* code_all, int32_t Bt, const float* lse, const int32_t* target,
                        int32_t row_offset, float inv_batch, float* dv_partial, void* stream) {
  int rc = check_batch(e, Bt);
  if (rc) return rc;
  if (!code_all || !lse || !target || !dv_partial) return fail(e, C2V_ERR_INVALID, "NULL argument");
  if (!e->has_grad) return fail(e, C2V_ERR_STATE, "gradients not bound (c2v_bind_grads)");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  const HeadSchedule hs = head_schedule(e, API_TARGET_BACKWARD, code_all);
  e->split_fwd = HEAD_SIMT;
  const umma::SoftmaxGradArgs g{lse, target, row_offset, inv_batch};
  SlabDesc slab;
  if (hs == HEAD_EXP_SLAB) {
    // the slab holds U = exp(s - c_b): patch the true-class elements and set the rows' factors; for a row that left the fp32
    // window the logits are computed again (gated) and rewritten with the global log-sum-exp, and its factor becomes 1
    float* S_lo = is_3x(e) ? wsp<float>(e, e->ws.S_lo) : nullptr;
    int* flag = wsp<int>(e, e->ws.slab_flag);
    {
      PhaseTimer pt(e, PH_XENT, st);
      C2V_LAUNCH(e, (expsum_finish_kernel<<<(Bt + 255) / 256, 256, 0, st>>>(wsp<float>(e, e->ws.S), S_lo, e->ws.ldS, e->dims.target_vocab,
                                                                            target, row_offset, wsp<float>(e, e->ws.true_logit), lse,
                                                                            inv_batch, Bt, wsp<float>(e, e->ws.rscale), flag)));
    }
    if ((rc = run_logits(e, st, code_all, Bt, LOGITS_STORE_LSE_GATED, LogitsArgs{nullptr, flag}))) return rc;
  }
  const float* v_dy;
  {
    PhaseTimer pt(e, PH_XENT, st);
    if ((rc = slab_to_p(e, st, hs, code_all, Bt, g, &slab, &v_dy, true))) return rc;
  }
  return target_grad_gemms(e, st, v_dy, Bt, dv_partial, slab);
}

int c2v_context_backward(c2v_engine* e, const int32_t* src, const int32_t* path, const int32_t* tgt, const float* mask,
                         int32_t B, float keep_prob, uint64_t seed, uint64_t step, const float* dropout_mask,
                         const float* dv, void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!src || !path || !tgt || !mask || !dv) return fail(e, C2V_ERR_INVALID, "NULL argument");
  if (!e->has_grad) return fail(e, C2V_ERR_STATE, "gradients not bound (c2v_bind_grads)");
  C2V_CUDA(e, cudaSetDevice(e->device));
  const Dropout dp = make_dropout(e->dims, keep_prob, seed, step, dropout_mask);
  ContextSource cs = make_source(e, src, path, tgt, B);
  return context_backward(e, (cudaStream_t)stream, cs, mask, B, dp, dv);
}

// ---- sampled softmax on a row-sharded target table (fully sharded schedule) ------------------------------
static bool rows_aligned(const void* p) { return ((uintptr_t)p % 16) == 0; }

int c2v_sampled_pack_rows(c2v_engine* e, const int32_t* sampled, int32_t S, const int32_t* target_all, int32_t Bt,
                          int32_t row_offset, float* neg_rows, float* true_rows, void* stream) {
  int rc = check_batch(e, Bt);
  if (rc) return rc;
  if (!sampled || !target_all || !neg_rows || !true_rows) return fail(e, C2V_ERR_INVALID, "NULL argument");
  if (S < 1 || S > kMaxSampled) return fail(e, C2V_ERR_INVALID, "number of sampled classes must be in [1, 1024]");
  if (!e->has_theta) return fail(e, C2V_ERR_STATE, "parameters not bound");
  if (!rows_aligned(neg_rows) || !rows_aligned(true_rows)) return fail(e, C2V_ERR_INVALID, "row buffers must be 16-byte aligned");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  const int D = e->dims.code_dim;
  const size_t n4 = (size_t)(S + Bt) * (D / 4);
  size_t blocks = (n4 + 255) / 256;
  if (blocks > (size_t)e->num_sms * 16) blocks = (size_t)e->num_sms * 16;
  PhaseTimer pt(e, PH_SAMPLED, st);
  C2V_LAUNCH(e, (sampled_pack_rows_kernel<<<(unsigned)blocks, 256, 0, st>>>(e->theta.tgt, e->dims.target_vocab, row_offset, sampled, S,
                                                                            target_all, Bt, D, neg_rows, true_rows)));
  return C2V_OK;
}

int c2v_sampled_target_step(c2v_engine* e, const float* code_vec, int32_t B, const int32_t* target, const int32_t* sampled,
                            int32_t S, const float* logq_true, const float* logq_sampled, const float* neg_rows,
                            const float* true_rows, float inv_batch, float* dv, float* g_true, float* g_neg,
                            float* loss_partial, void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!code_vec || !target || !sampled || !logq_true || !logq_sampled || !neg_rows || !true_rows || !dv || !g_true || !g_neg ||
      !loss_partial)
    return fail(e, C2V_ERR_INVALID, "NULL argument");
  if (S < 1 || S > kMaxSampled) return fail(e, C2V_ERR_INVALID, "number of sampled classes must be in [1, 1024]");
  if (!rows_aligned(code_vec) || !rows_aligned(neg_rows) || !rows_aligned(true_rows))
    return fail(e, C2V_ERR_INVALID, "code vectors and row buffers must be 16-byte aligned");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  const int D = e->dims.code_dim;
  float* loss_b = wsp<float>(e, e->ws.loss_b);
  float* dl = wsp<float>(e, e->ws.dl);
  PhaseTimer pt(e, PH_SAMPLED, st);
  const size_t smem = ((size_t)D + S + 1) * sizeof(float);
  C2V_LAUNCH(e, (sampled_softmax_rows_fwd_kernel<<<B, kSampledThreads, smem, st>>>(code_vec, true_rows, neg_rows, target, sampled, S,
                                                                                   logq_true, logq_sampled, D, inv_batch, loss_b, dl,
                                                                                   dv)));
  C2V_LAUNCH(e, (loss_reduce_kernel<<<1, 256, 0, st>>>(loss_b, B, inv_batch, loss_partial)));
  C2V_LAUNCH(e, (sampled_true_grad_kernel<<<B, kSampledThreads, 0, st>>>(code_vec, dl, S, D, g_true)));
  C2V_LAUNCH(e, (sampled_neg_grad_kernel<<<dim3(S, (D + 31) / 32), kNegGradWarps * 32, 0, st>>>(code_vec, dl, B, S, D, g_neg)));
  return C2V_OK;
}

int c2v_sampled_target_fold(c2v_engine* e, const float* g_true_all, const float* g_neg_all, int32_t world,
                            const int32_t* target_all, int32_t Bt, const int32_t* sampled, int32_t S, int32_t row_offset,
                            const float* loss_parts, float* loss_out, void* stream) {
  int rc = check_batch(e, Bt);
  if (rc) return rc;
  if (!g_true_all || !g_neg_all || !target_all || !sampled || !loss_parts || !loss_out)
    return fail(e, C2V_ERR_INVALID, "NULL argument");
  if (S < 1 || S > kMaxSampled) return fail(e, C2V_ERR_INVALID, "number of sampled classes must be in [1, 1024]");
  if (world < 1 || world > kMaxShards) return fail(e, C2V_ERR_INVALID, "world out of range");
  if (!e->has_grad) return fail(e, C2V_ERR_STATE, "gradients not bound (c2v_bind_grads)");
  const int D = e->dims.code_dim;
  if (D > kFoldThreads * kFoldCols) return fail(e, C2V_ERR_INVALID, "code_dim too large for the fold");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  const int Yl = e->dims.target_vocab;
  PhaseTimer pt(e, PH_SAMPLED, st);
  // the block may hold a full-softmax step's gradient (or a stale one after a fused Adam): every row is written here
  C2V_CUDA(e, cudaMemsetAsync(e->grad.tgt, 0, (size_t)Yl * D * 4, st));
  C2V_LAUNCH(e, (sampled_target_fold_kernel<<<Bt + S, kFoldThreads, 0, st>>>(g_true_all, g_neg_all, world, target_all, Bt, sampled, S,
                                                                             D, row_offset, Yl, e->grad.tgt)));
  C2V_LAUNCH(e, (sum_in_order_kernel<<<1, 1, 0, st>>>(loss_parts, world, loss_out)));
  return C2V_OK;
}

int c2v_sync_tables(c2v_engine* e, void* stream) {
  if (!e) return C2V_ERR_INVALID;
  C2V_CUDA(e, cudaSetDevice(e->device));
  return flush_rows(e, (cudaStream_t)stream);
}

int c2v_set_event(c2v_engine* e, const char* name, void* cuda_event) {
  if (!e || !name) return C2V_ERR_INVALID;
  if (!strcmp(name, "target_grads_ready")) { e->ev_tgt_ready = (cudaEvent_t)cuda_event; return C2V_OK; }
  return fail(e, C2V_ERR_INVALID, std::string("unknown event: ") + name);
}

int c2v_adam_step_range(c2v_engine* e, float* theta, float* grad, float* m, float* v, size_t count, float lr,
                        float beta1, float beta2, float eps, int64_t t, int32_t zero_grad, void* stream) {
  if (!e) return C2V_ERR_INVALID;
  if (!theta || !grad || !m || !v) return fail(e, C2V_ERR_INVALID, "NULL argument");
  if (count % 4 || ((uintptr_t)theta | (uintptr_t)grad | (uintptr_t)m | (uintptr_t)v) % 16)
    return fail(e, C2V_ERR_INVALID, "slice must be a multiple of 4 floats and 16-byte aligned");
  if (t < 1) return fail(e, C2V_ERR_INVALID, "Adam step count t must be >= 1");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  const float lr_t = (float)((double)lr * sqrt(1.0 - pow((double)beta2, (double)t)) / (1.0 - pow((double)beta1, (double)t)));
  const size_t n4 = count / 4;
  if (n4 == 0) return C2V_OK;
  size_t blocks = (n4 + 255) / 256;
  if (blocks > (size_t)e->num_sms * 16) blocks = (size_t)e->num_sms * 16;
  PhaseTimer pt(e, PH_ADAM, st);
  C2V_LAUNCH(e, (adam_kernel<<<(unsigned)blocks, 256, 0, st>>>(theta, grad, m, v, n4, lr_t, beta1, beta2, eps,
                                                               zero_grad ? 1 : 0)));
  return C2V_OK;
}

int c2v_train_batch_host(c2v_engine* e, const int32_t* h_src, const int32_t* h_path, const int32_t* h_tgt,
                         const float* h_mask, const int32_t* h_target, int32_t B, float keep_prob, uint64_t seed,
                         int64_t t, float lr, float beta1, float beta2, float eps, float* h_loss, void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!h_src || !h_path || !h_tgt || !h_mask || !h_target || !h_loss) return fail(e, C2V_ERR_INVALID, "NULL argument");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t nb = (size_t)B * e->dims.max_contexts * 4;
  int32_t* src = wsp<int32_t>(e, e->ws.st_src);
  int32_t* pth = wsp<int32_t>(e, e->ws.st_pth);
  int32_t* tgt = wsp<int32_t>(e, e->ws.st_tgt);
  float* mask = wsp<float>(e, e->ws.st_mask);
  int32_t* target = wsp<int32_t>(e, e->ws.st_target);
  float* loss = wsp<float>(e, e->ws.loss);
  C2V_CUDA(e, cudaMemcpyAsync(src, h_src, nb, cudaMemcpyHostToDevice, st));
  C2V_CUDA(e, cudaMemcpyAsync(pth, h_path, nb, cudaMemcpyHostToDevice, st));
  C2V_CUDA(e, cudaMemcpyAsync(tgt, h_tgt, nb, cudaMemcpyHostToDevice, st));
  C2V_CUDA(e, cudaMemcpyAsync(mask, h_mask, nb, cudaMemcpyHostToDevice, st));
  C2V_CUDA(e, cudaMemcpyAsync(target, h_target, (size_t)B * 4, cudaMemcpyHostToDevice, st));
  if (e->fuse_tgt && (rc = c2v_arm_target_adam(e, lr, beta1, beta2, eps, t))) return rc;
  // the Adam step count doubles as the dropout stream position
  if ((rc = train_step_impl(e, st, src, pth, tgt, mask, target, B, keep_prob, seed, (uint64_t)t, nullptr, loss))) return rc;
  if ((rc = adam_impl(e, st, lr, beta1, beta2, eps, t))) return rc;
  C2V_CUDA(e, cudaMemcpyAsync(h_loss, loss, 4, cudaMemcpyDeviceToHost, st));
  C2V_CUDA(e, cudaStreamSynchronize(st));
  return C2V_OK;
}

int c2v_train_batch_async(c2v_engine* e, const int32_t* h_src, const int32_t* h_path, const int32_t* h_tgt, const float* h_mask,
                          const int32_t* h_target, int32_t B, float keep_prob, uint64_t seed, int64_t t, float lr, float beta1,
                          float beta2, float eps, float* h_loss, void* upload_done_event, void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!h_src || !h_path || !h_tgt || !h_mask || !h_target || !h_loss) return fail(e, C2V_ERR_INVALID, "NULL argument");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  const int i = (int)(e->async_n++ & 1);
  const size_t nb = (size_t)B * e->dims.max_contexts * 4;
  int32_t* src = wsp<int32_t>(e, i ? e->ws.sb_src : e->ws.st_src);
  int32_t* pth = wsp<int32_t>(e, i ? e->ws.sb_pth : e->ws.st_pth);
  int32_t* tgt = wsp<int32_t>(e, i ? e->ws.sb_tgt : e->ws.st_tgt);
  float* mask = wsp<float>(e, i ? e->ws.sb_mask : e->ws.st_mask);
  int32_t* target = wsp<int32_t>(e, i ? e->ws.sb_target : e->ws.st_target);
  float* loss = wsp<float>(e, e->ws.loss) + 1 + i;          // one device slot per buffer: the previous step's read-back may be in flight
  // upload on the copy stream, behind the step that last read this staging set; the step waits for the upload only
  if (e->used_valid[i]) C2V_CUDA(e, cudaStreamWaitEvent(e->copy, e->ev_used[i], 0));
  C2V_CUDA(e, cudaMemcpyAsync(src, h_src, nb, cudaMemcpyHostToDevice, e->copy));
  C2V_CUDA(e, cudaMemcpyAsync(pth, h_path, nb, cudaMemcpyHostToDevice, e->copy));
  C2V_CUDA(e, cudaMemcpyAsync(tgt, h_tgt, nb, cudaMemcpyHostToDevice, e->copy));
  C2V_CUDA(e, cudaMemcpyAsync(mask, h_mask, nb, cudaMemcpyHostToDevice, e->copy));
  C2V_CUDA(e, cudaMemcpyAsync(target, h_target, (size_t)B * 4, cudaMemcpyHostToDevice, e->copy));
  C2V_CUDA(e, cudaEventRecord(e->ev_h2d[i], e->copy));
  if (upload_done_event) C2V_CUDA(e, cudaEventRecord((cudaEvent_t)upload_done_event, e->copy));
  C2V_CUDA(e, cudaStreamWaitEvent(st, e->ev_h2d[i], 0));
  if (e->fuse_tgt && (rc = c2v_arm_target_adam(e, lr, beta1, beta2, eps, t))) return rc;
  if ((rc = train_step_impl(e, st, src, pth, tgt, mask, target, B, keep_prob, seed, (uint64_t)t, nullptr, loss))) return rc;
  if ((rc = adam_impl(e, st, lr, beta1, beta2, eps, t))) return rc;
  C2V_CUDA(e, cudaMemcpyAsync(h_loss, loss, 4, cudaMemcpyDeviceToHost, st));
  C2V_CUDA(e, cudaEventRecord(e->ev_used[i], st));
  e->used_valid[i] = true;
  return C2V_OK;
}

int c2v_predict_batch_host(c2v_engine* e, const int32_t* h_src, const int32_t* h_path, const int32_t* h_tgt,
                           const float* h_mask, int32_t B, int32_t normalize, int32_t* h_topk_idx, float* h_topk_val,
                           float* h_code_vec, float* h_attn, void* stream) {
  int rc = check_batch(e, B);
  if (rc) return rc;
  if (!h_src || !h_path || !h_tgt || !h_mask || !h_topk_idx || !h_topk_val) return fail(e, C2V_ERR_INVALID, "NULL argument");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t nb = (size_t)B * e->dims.max_contexts * 4;
  int32_t* src = wsp<int32_t>(e, e->ws.st_src);
  int32_t* pth = wsp<int32_t>(e, e->ws.st_pth);
  int32_t* tgt = wsp<int32_t>(e, e->ws.st_tgt);
  float* mask = wsp<float>(e, e->ws.st_mask);
  float* code = wsp<float>(e, e->ws.st_code);
  float* attn = wsp<float>(e, e->ws.st_attn);
  int32_t* tki = wsp<int32_t>(e, e->ws.st_topk_idx);
  float* tkv = wsp<float>(e, e->ws.st_topk_val);
  C2V_CUDA(e, cudaMemcpyAsync(src, h_src, nb, cudaMemcpyHostToDevice, st));
  C2V_CUDA(e, cudaMemcpyAsync(pth, h_path, nb, cudaMemcpyHostToDevice, st));
  C2V_CUDA(e, cudaMemcpyAsync(tgt, h_tgt, nb, cudaMemcpyHostToDevice, st));
  C2V_CUDA(e, cudaMemcpyAsync(mask, h_mask, nb, cudaMemcpyHostToDevice, st));
  const Dropout dp = make_dropout(e->dims, 1.0f, 0, 0, nullptr);
  if ((rc = forward_impl(e, st, src, pth, tgt, mask, B, dp, code, attn))) return rc;
  if ((rc = topk_impl(e, st, code, B, tki, tkv, normalize))) return rc;
  const int Y = e->dims.target_vocab;
  const int k = e->dims.top_k < Y ? e->dims.top_k : Y;
  C2V_CUDA(e, cudaMemcpyAsync(h_topk_idx, tki, (size_t)B * k * 4, cudaMemcpyDeviceToHost, st));
  C2V_CUDA(e, cudaMemcpyAsync(h_topk_val, tkv, (size_t)B * k * 4, cudaMemcpyDeviceToHost, st));
  if (h_code_vec) C2V_CUDA(e, cudaMemcpyAsync(h_code_vec, code, (size_t)B * e->dims.code_dim * 4, cudaMemcpyDeviceToHost, st));
  if (h_attn) C2V_CUDA(e, cudaMemcpyAsync(h_attn, attn, nb, cudaMemcpyDeviceToHost, st));
  C2V_CUDA(e, cudaStreamSynchronize(st));
  return C2V_OK;
}

int c2v_selftest_gemm(c2v_engine* e, int32_t a_mn, int32_t b_mn, int32_t bn, int32_t M, int32_t N, int32_t K,
                      int32_t splits, const float* A, size_t lda, const float* Bm, size_t ldb, float* C, size_t ldc,
                      void* stream) {
  return c2v_selftest_gemm3(e, a_mn, b_mn, bn, M, N, K, splits, A, nullptr, lda, Bm, nullptr, ldb, C, ldc, stream);
}

int c2v_selftest_gemm3(c2v_engine* e, int32_t a_mn, int32_t b_mn, int32_t bn, int32_t M, int32_t N, int32_t K,
                       int32_t splits, const float* A, const float* A_lo, size_t lda, const float* Bm, const float* B_lo,
                       size_t ldb, float* C, size_t ldc, void* stream) {
  if (!e || !A || !Bm || !C) return C2V_ERR_INVALID;
  if ((A_lo != nullptr) != (B_lo != nullptr)) return fail(e, C2V_ERR_INVALID, "3xTF32 needs the low parts of both operands");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  umma::Operand opA{A, lda, a_mn != 0, A_lo};
  umma::Operand opB{Bm, ldb, b_mn != 0, B_lo};
  if (!umma::operand_ok(opA) || !umma::operand_ok(opB)) return fail(e, C2V_ERR_INVALID, "operand not TMA-compatible");
  umma::EpiStore ep{C, ldc, (size_t)M * ldc};
  if (bn != 192 && bn != 256) return fail(e, C2V_ERR_INVALID, "bn must be 192 or 256");
  C2V_LAUNCH(e, C2V_CUDA(e, (umma::launch(st, M, N, K, splits, opA, opB, ep, e->num_sms))));
  return umma::effective_splits(K, splits);
}

int c2v_selftest_gemm_bt(c2v_engine* e, int32_t M, int32_t N, int32_t K, const float* A, size_t lda, const float* Bm, size_t ldb,
                         float* C, size_t ldc, float* BT, size_t ldbt, void* stream) {
  if (!e || !A || !Bm || !C || !BT) return C2V_ERR_INVALID;
  C2V_CUDA(e, cudaSetDevice(e->device));
  const umma::Operand opA{A, lda, false}, opB{Bm, ldb, false};
  if (!umma::operand_ok(opA) || !umma::operand_ok(opB)) return fail(e, C2V_ERR_INVALID, "operand not TMA-compatible");
  const umma::EpiStore ep{C, ldc, 0};
  C2V_LAUNCH(e, C2V_CUDA(e, (umma::launch_cfg<false, false, umma::EpiStore, umma::AXNone, true>((cudaStream_t)stream, M, N, K, 1, opA, opB,
                                                                                                ep, e->num_sms, umma::AXNone{},
                                                                                                umma::BTransposed{BT, nullptr, ldbt}))));
  return C2V_OK;
}

int c2v_selftest_split(c2v_engine* e, const float* x, float* hi, float* lo, size_t count, void* stream) {
  if (!e || !x || !hi || !lo) return C2V_ERR_INVALID;
  if (count % 4 || ((uintptr_t)x | (uintptr_t)hi | (uintptr_t)lo) % 16) return fail(e, C2V_ERR_INVALID, "count % 4 and 16-byte alignment");
  C2V_CUDA(e, cudaSetDevice(e->device));
  size_t blocks = (count / 4 + 255) / 256;
  if (blocks > (size_t)e->num_sms * 16) blocks = (size_t)e->num_sms * 16;
  if (blocks < 1) blocks = 1;
  C2V_LAUNCH(e, (split_tf32_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, hi, lo, count / 4)));
  return C2V_OK;
}

int c2v_selftest_transpose(c2v_engine* e, const float* x, int32_t rows, int32_t cols, float* xT, float* xT_lo, size_t ldT,
                           void* stream) {
  if (!e || !x || !xT) return C2V_ERR_INVALID;
  if (rows < 1 || cols < 1 || ldT < (size_t)rows || cols > 65535 * 32) return fail(e, C2V_ERR_INVALID, "bad size");
  C2V_CUDA(e, cudaSetDevice(e->device));
  const dim3 grid((unsigned)((rows + 31) / 32), (unsigned)((cols + 31) / 32));
  cudaStream_t st = (cudaStream_t)stream;
  if (xT_lo) C2V_LAUNCH(e, (transpose_kernel<true><<<grid, 256, 0, st>>>(x, rows, cols, xT, xT_lo, ldT, nullptr, nullptr)));
  else C2V_LAUNCH(e, (transpose_kernel<false><<<grid, 256, 0, st>>>(x, rows, cols, xT, nullptr, ldT, nullptr, nullptr)));
  return C2V_OK;
}

int c2v_selftest_target_t(const c2v_engine* e, int32_t lo, size_t* offset, size_t* ld) {
  if (!e || !offset || !ld) return C2V_ERR_INVALID;
  *offset = lo ? e->ws.tgtT_lo : e->ws.tgtT;
  *ld = e->ws.ldS;
  return C2V_OK;
}

int c2v_selftest_row_sum(c2v_engine* e, int32_t table_id, const int32_t* rows, const float* vals, int32_t count, float* out,
                         void* stream) {
  if (!e || !rows || !vals || !out) return C2V_ERR_INVALID;
  if (!e->wbase) return fail(e, C2V_ERR_STATE, "workspace not bound (c2v_bind_workspace)");
  if (table_id != 0 && table_id != 1) return fail(e, C2V_ERR_INVALID, "table_id must be 0 (token table) or 1 (path table)");
  if (count < 0 || (int64_t)count > 3ll * e->dims.max_batch * e->dims.max_contexts)
    return fail(e, C2V_ERR_INVALID, "count must be in [0, 3 * max_batch * max_contexts]");
  if (((uintptr_t)vals | (uintptr_t)out) % 16) return fail(e, C2V_ERR_INVALID, "vals and out must be 16-byte aligned");
  if ((int64_t)e->dims.token_vocab + e->dims.path_vocab >= INT32_MAX)
    return fail(e, C2V_ERR_UNSUPPORTED, "token_vocab + path_vocab must be below 2^31");
  C2V_CUDA(e, cudaSetDevice(e->device));
  const c2v_dims& d = e->dims;
  const DetDest dst{out, out, d.token_vocab, d.embed_dim};
  return det_row_sums(e, (cudaStream_t)stream, DetListKeys{rows, table_id ? d.token_vocab : 0}, count,
                      (uint32_t)(d.token_vocab + d.path_vocab), DetListContrib{vals, d.embed_dim}, dst);
}

int c2v_selftest_exchange_push(c2v_engine* e, const int32_t* tok_rows, const float* tok_vals, int32_t n_tok,
                               const int32_t* path_rows, const float* path_vals, int32_t n_path, void* stream) {
  if (!e || n_tok < 0 || n_path < 0) return C2V_ERR_INVALID;
  if ((n_tok && (!tok_rows || !tok_vals)) || (n_path && (!path_rows || !path_vals))) return fail(e, C2V_ERR_INVALID, "NULL list");
  if (!e->wbase) return fail(e, C2V_ERR_STATE, "workspace not bound (c2v_bind_workspace)");
  if (!ordered_route(e)) return fail(e, C2V_ERR_STATE, "set ordered_exchange and bind row-sharded tables over more than one rank first");
  if (e->inbox.world < 2) return fail(e, C2V_ERR_STATE, "no scatter inbox bound (c2v_bind_scatter_inbox)");
  if ((int64_t)n_tok + n_path > 3ll * e->dims.max_batch * e->dims.max_contexts)
    return fail(e, C2V_ERR_INVALID, "n_tok + n_path must be at most 3 * max_batch * max_contexts");
  if (((uintptr_t)tok_vals | (uintptr_t)path_vals) % 16) return fail(e, C2V_ERR_INVALID, "tok_vals and path_vals must be 16-byte aligned");
  C2V_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  // one [n_tok + n_path, d] list of contributions, in the dX' region (it holds 3 * max_batch * max_contexts rows of d)
  const size_t d = (size_t)e->dims.embed_dim;
  float* vals = wsp<float>(e, e->ws.dXg);
  if (n_tok) C2V_CUDA(e, cudaMemcpyAsync(vals, tok_vals, n_tok * d * 4, cudaMemcpyDeviceToDevice, st));
  if (n_path) C2V_CUDA(e, cudaMemcpyAsync(vals + n_tok * d, path_vals, n_path * d * 4, cudaMemcpyDeviceToDevice, st));
  return exchange_push(e, st, ExchangeListKeys{tok_rows, path_rows, n_tok, exchange_key_map(e)}, n_tok + n_path,
                       DetListContrib{vals, (int)d});
}

int64_t c2v_launch_count(const c2v_engine* e) { return e ? e->launches : 0; }

int c2v_phase_count(void) { return PH_COUNT; }

const char* c2v_phase_name(int phase) { return (phase >= 0 && phase < PH_COUNT) ? kPhaseNames[phase] : ""; }

int c2v_phase_stats(c2v_engine* e, int phase, double* total_ms, int64_t* count, int reset) {
  if (!e || phase < 0 || phase >= PH_COUNT) return C2V_ERR_INVALID;
  C2V_CUDA(e, cudaSetDevice(e->device));
  PhaseLog& L = e->phase[phase];
  if (!L.pending.empty()) C2V_CUDA(e, cudaDeviceSynchronize());
  for (auto& ev : L.pending) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ev.first, ev.second) == cudaSuccess) { L.total_ms += ms; L.count++; }
    L.free_list.push_back(ev);
  }
  L.pending.clear();
  if (total_ms) *total_ms = L.total_ms;
  if (count) *count = L.count;
  if (reset) { L.total_ms = 0.0; L.count = 0; }
  return C2V_OK;
}

}  // extern "C"
