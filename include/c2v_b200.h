/*
 * c2v_b200.h -- C ABI of the H100-native (sm_90a) path-attention engine (libc2v_b200.so).
 *
 * This is the drop-in boundary for code2vec's ONE hot path.  The reference (tech-srl/code2vec)
 * has no FFI of its own: its seam is the Python ABC Code2VecModelBase (model_base.py:37-182)
 * whose TensorFlow backend runs the whole path inside sess.run() calls.  Each entry point below
 * names the reference statement(s) it replaces (file:line relative to the reference root), so a
 * maintainer can bind it from a third backend (`--framework b200`, see INTEGRATION.md).
 *
 * Conventions
 *   - plain C, no CUDA / torch types: device pointers are `void*`/`float*`/`int32_t*` holding
 *     device addresses, a stream is the `cudaStream_t` value passed as `void*` (NULL = default).
 *   - every function returns 0 (C2V_OK) or a negative c2v_status; the message of the last
 *     failure is kept per engine (c2v_last_error).  Nothing throws across the boundary.
 *   - the caller owns all big buffers (parameters, gradients, Adam slots, workspace) -- in the
 *     Python backend they are torch tensors used purely as storage.  The engine allocates
 *     nothing on the device after c2v_create.
 *   - all calls are asynchronous w.r.t. the host on `stream`, except the *_host entry points,
 *     which synchronise the stream before returning because they hand results back to the host.
 *   - one host thread per engine at a time; engines are independent.
 *   - layouts: row-major, float32 parameters, int32 indices, float32 0/1 mask -- the dtypes the
 *     reference reader emits (path_context_reader.py:32-44,214; vocabularies.py:112).
 */
#ifndef C2V_B200_H_
#define C2V_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define C2V_ABI_VERSION 1

typedef struct c2v_engine c2v_engine;

typedef enum c2v_status {
  C2V_OK = 0,
  C2V_ERR_INVALID = -1,      /* bad argument (NULL, size out of range, unsupported dims)   */
  C2V_ERR_CUDA = -2,         /* a CUDA runtime call or kernel launch failed                */
  C2V_ERR_STATE = -3,        /* call order violated (e.g. train step before binding grads) */
  C2V_ERR_UNSUPPORTED = -4   /* valid request this build cannot serve                      */
} c2v_status;

/* Shapes of the model (config.py:60-68; vocab sizes include the special words,
 * vocabularies.py:51-55).  code_dim is CODE_VECTOR_SIZE (= 3*embed_dim by default). */
typedef struct c2v_dims {
  int32_t token_vocab;   /* T: rows of WORDS_VOCAB          (tensorflow_model.py:206-209) */
  int32_t path_vocab;    /* P: rows of PATHS_VOCAB          (tensorflow_model.py:217-220) */
  int32_t target_vocab;  /* Y: rows of TARGET_WORDS_VOCAB   (tensorflow_model.py:210-213) */
  int32_t embed_dim;     /* d: TOKEN/PATH_EMBEDDINGS_SIZE, multiple of 4                  */
  int32_t code_dim;      /* D: CODE_VECTOR_SIZE, multiple of 4, <= 1024                   */
  int32_t max_contexts;  /* C: MAX_CONTEXTS                                               */
  int32_t max_batch;     /* largest batch any call will pass                              */
  int32_t top_k;         /* TOP_K_WORDS_CONSIDERED_DURING_PREDICTION (<= 64)              */
} c2v_dims;

/* The five variables of the model, in the order the reference creates them
 * (tensorflow_model.py:32-36,205-220,249-250).  Used for parameters, gradients and Adam slots.
 *   tok  [T, d]   WORDS_VOCAB            path [P, d]   PATHS_VOCAB
 *   tgt  [Y, D]   TARGET_WORDS_VOCAB     W    [3d, D]  TRANSFORM          a [D] ATTENTION */
typedef struct c2v_tensors {
  float* tok;
  float* path;
  float* tgt;
  float* W;
  float* a;
} c2v_tensors;

/* Arithmetic of the three big matrix products (projection, logits, their gradients).
 *   C2V_MATH_FP32  : fp32 FFMA on the SIMT pipe -- the reference's own arithmetic class
 *                    (cuBLAS/Eigen SGEMM); used for bit-level top-k parity.
 *   C2V_MATH_TF32  : wgmma tf32 (fp32 storage, 10-bit mantissa operands, fp32
 *                    accumulate in registers) -- what TensorFlow itself runs on Ampere+ GPUs.
 *   C2V_MATH_3XTF32: the same tensor-core kernels at fp32-equivalent accuracy: every operand is
 *                    split into tf32 high and low parts (x = hi + lo up to 2^-22 |x|) and a product
 *                    is issued as a_lo.b_hi + a_hi.b_lo + a_hi.b_hi into the same fp32 register
 *                    accumulator (the dropped a_lo.b_lo term is O(2^-22) relative); tanh / exp in the
 *                    epilogues use the correctly rounded library forms.  The reference's arithmetic
 *                    class (fp32 tf.matmul, tensorflow_model.py:226,252,297) on tensor cores. */
typedef enum c2v_math_mode { C2V_MATH_FP32 = 0, C2V_MATH_TF32 = 1, C2V_MATH_3XTF32 = 2 } c2v_math_mode;

int c2v_abi_version(void);

/* Message of the last failed call on `e`; with e == NULL, of the last failed c2v_create /
 * c2v_workspace_bytes on this thread.  Never NULL. */
const char* c2v_last_error(const c2v_engine* e);

/* Bytes of device scratch the engine needs for `dims` (activations kept for the backward pass,
 * the [B, Y] logits slab, split-K partials, host-API staging).  0 on invalid dims. */
size_t c2v_workspace_bytes(const c2v_dims* dims);

/* Create an engine for CUDA device `device`.  Replaces Code2VecModel.__init__'s
 * tf.compat.v1.Session() (tensorflow_model.py:19-38). */
int c2v_create(const c2v_dims* dims, int device, c2v_engine** out);

/* Replaces close_session() (tensorflow_model.py:439-440).  NULL is a no-op. */
void c2v_destroy(c2v_engine* e);

int c2v_bind_workspace(c2v_engine* e, void* dev_ptr, size_t bytes);   /* >= c2v_workspace_bytes, 256-B aligned */
int c2v_bind_params(c2v_engine* e, const c2v_tensors* theta);         /* tf.get_variable x5, :205-220,249-250   */
int c2v_bind_grads(c2v_engine* e, const c2v_tensors* grads);          /* autodiff outputs of minimize(), :232   */
int c2v_bind_adam_state(c2v_engine* e, const c2v_tensors* m, const c2v_tensors* v);  /* Adam slots, :232       */

/* Options: "math_mode" (c2v_math_mode), "deterministic" (0/1, default 0, may change between steps: with 1 a train step's
 * results depend only on its inputs, seeds and options -- not on scheduling, streams or the run -- on the same build and
 * device type.  Every other reduction of a step is fixed-order already; this option replaces the two that use float
 * atomics.  Embedding gradients: for a gradient row, the unmasked entries e = 3 n + seg that reference it (token table:
 * seg 0 = source, 2 = target; path table: seg 1) are listed in increasing e; entry e contributes exactly what the atomic
 * scatter adds (dX'[n, seg d : (seg+1) d] x dropout multiplier x grad scale); the list is cut into consecutive chunks of
 * K = 32 entries starting at the row's first entry, each chunk is summed left to right from +0.0f, and the chunk sums are
 * added left to right from +0.0f.  Sampled softmax (c2v_sampled_train_step): a target row's gradient is, from +0.0f and
 * left to right, its true-row terms dl[b,0] v_b in b order, then for each sampled position s holding the row (in s order)
 * the sums over b of dl[b,1+s] v_b in chunks of 64 examples, chunk by chunk.  Refused (C2V_ERR_UNSUPPORTED) while the
 * embedding tables are row-sharded over more than one rank (c2v_bind_table_shards, world > 1; a scatter inbox can only be
 * bound on top of that) -- their cross-rank red.adds and inbox folds stay order-free -- and binding such shards while it
 * is set fails the same way -- unless "ordered_exchange" is set.  The order in which NCCL reduces
 * the gradients of data-parallel schedules is outside this guarantee), "ordered_exchange" (0/1, default 0; no effect on
 * one rank.  With 1, a train step or c2v_context_backward on tables row-sharded over W > 1 ranks sends embedding gradients
 * through the scatter inbox in a fixed order, in every math mode, and "deterministic" is accepted on such tables: each
 * sender s reduces its own entries of a row to ONE sum R_s in the order "deterministic" documents and pushes one (local
 * row, R_s) record per distinct row, sorted by row, and c2v_apply_scatter_inbox stores G, where G = +0.0f and then
 * G = fl(G + R_s) for s = 0 .. W-1, skipping senders without an entry for the row (the shard's gradient rows must be zero
 * before the step; rows nobody references are not written).  Same inputs, seeds, options, build and world size then give
 * the same bits; a single engine on the global batch associates differently.  Needs c2v_bind_scatter_inbox: a backward
 * pass without one fails with C2V_ERR_STATE.  Cannot be cleared (C2V_ERR_UNSUPPORTED) while "deterministic" is set on
 * tables sharded over more than one rank; refused unless token_vocab + path_vocab + 16 < 2^31), "ordered_exchange_rows"
 * (read-only: the records this rank pushed in its last ordered exchange, summed over owners; synchronises), "cta_pair"
 * (0, 1 or 2, default 2: accepted for ABI compatibility
 * (it once selected CTA-pair GEMMs); the sm_90a GEMM has no CTA-pair form and ignores it), "dy_late" (where the target-table gradient GEMM dY = P^T.v -- with the
 * target table's Adam step in its epilogue when armed -- runs: 0 = right after dv on the caller's
 * stream, "target_grads_ready" fires earliest; 1 = default: inside the context backward pass, next
 * to the embedding scatter-add; 2 = on an engine-owned stream right after dv, joined before the
 * step returns.  All three measure within 1 % of each other on one GPU: the persistent GEMM CTAs
 * fill the register file, so kernels on other streams mostly wait for them), "profile" (0/1: per-phase
 * CUDA-event timing, read with c2v_phase_stats), "lazy_adam" (0/1, single-GPU replicated tables:
 * the dense TF1 Adam update of an embedding row is deferred -- its gradient stays in the bound
 * gradient table -- and replayed bit-exactly (one step with that gradient, then the zero-gradient
 * steps) when a later batch references the row; same results as the dense update, one pass over
 * the batch's rows per step instead of 9 GB of traffic.  While it is on, the token / path gradient
 * tables are engine state (deferred steps), every c2v_train_step must be followed by
 * c2v_adam_step with consecutive t, and c2v_sync_tables brings every row up to date),
 * "adam_step_count" (the number of Adam steps already applied: optimizer reset / restore),
 * "grad_scale_inverse" (n: embedding scatter-adds are scaled by 1/n), "fuse_target_adam" (0/1,
 * default 0: c2v_train_batch_host arms c2v_arm_target_adam itself), "target_adam_fused_step"
 * (read: the step count whose target-table update the dY epilogue has already applied, 0 = none;
 * writing 0 acknowledges it for callers that drive c2v_adam_step_range themselves),
 * "early_catchup_count" (read-only: how many train steps used a c2v_hint_next_batch hint),
 * "adam_rows_occupancy" (4 or 5 resident blocks per SM for the lazy-Adam row pass; default 4),
 * "adam_sweep_period" (R, default 32, 0 = off: with lazy_adam every c2v_adam_step also brings rows
 * [rows*(t mod R)/R, rows*(t mod R + 1)/R) of each lazily updated table up to date, so that no row is
 * ever more than R steps behind -- this bounds the replay a rarely referenced row costs when a batch
 * finally reads it, and the cost of c2v_sync_tables, whatever the index distribution; results are
 * unchanged, the deferred steps are only applied earlier), "adam_rest_shortcut" (0/1, default 1: a row's
 * zero-gradient replay stops dividing / taking square roots once an update no longer changes any element of
 * the row -- updates shrink monotonically from there, so the parameters provably stay put and only the
 * slots keep decaying; bit-identical to the full replay for 0 < beta1 <= 0.95 and 0.99 <= beta2 < 1, and
 * not applied outside that range), "exp_slab" (0/1, default 1; tensor-core math modes, single-GPU full-softmax
 * train step): the logits GEMM's epilogue writes U = exp(logit - true-class logit) instead of the logits, one element
 * per row is patched and the softmax's 1 / sum is applied as a per-example factor by the two target-side gradient
 * GEMMs, so no pass re-reads the [B, Y] slab to normalise it; a step in which some row's largest U leaves the fp32
 * window [1e-26, 1e30], or some row's scaled code vector (the factor times v_b, dY's operand) has its largest
 * element below 2^-112 (subnormal elements would lose most of their bits on the tensor cores), is redone on the
 * device as the two-pass schedule (logits stored, then rewritten) -- read-only
 * "exp_slab_fallbacks" counts those steps (the read synchronises the device), "sort_peer_access" (row-sharded
 * tables over peer memory: 0 never, 1 = default: when a table exceeds 2 GB, 2 always -- the step's row indices are
 * counting-sorted by (owner, 2 MB page) before the peer gather / scatter-add).
 * Experimental schedules, all correct, all 0 by default (DESIGN.md sections
 * 4.6 - 4.8): "fuse_gather" (the gather feeds the context GEMM's shared-memory stages directly), "fuse_softmax_grad"
 * (dv / dY turn logits into dL/dlogits as their A tiles land; tf32 mode), "recompute_logits" (the logits GEMM runs
 * twice instead of storing logits), "adam_epilogue_prefetch" (the dY GEMM's Adam epilogue prefetches the (theta, m, v)
 * lines of its next tile into L2). */
int c2v_set_option(c2v_engine* e, const char* key, int64_t value);
int c2v_get_option(const c2v_engine* e, const char* key, int64_t* value);

/* _calculate_weighted_contexts(..., is_evaluating=True)  (tensorflow_model.py:236-265):
 * three gathers, concat, tanh(x.W), attention score, log-mask, softmax over the bag, weighted
 * sum.  src/path/tgt/mask: device [B, C].  code_vec: device [B, D].  attn: device [B, C] or
 * NULL.  A bag with no valid context yields NaN (as tf.nn.softmax of all -inf does). */
int c2v_forward(c2v_engine* e, const int32_t* src, const int32_t* path, const int32_t* tgt,
                const float* mask, int32_t B, float* code_vec, float* attn, void* stream);

/* scores = code_vec . TARGET_WORDS_VOCAB^T ; tf.nn.top_k(scores, k) sorted descending, ties to
 * the lower index (tensorflow_model.py:297-306).  normalize: 0 = raw scores (evaluate); 1 =
 * softmax over the k values (TF backend's predict, :305-306); 2 = probabilities of the softmax
 * over the whole target vocabulary (Keras backend: Dense(softmax) then top_k,
 * keras_model.py:69-70, keras_topk_word_predictions_layer.py:30-35).
 * idx: device int32 [B, k]; val: device float [B, k]. */
int c2v_topk(c2v_engine* e, const float* code_vec, int32_t B, int32_t* idx, float* val,
             int32_t normalize, void* stream);

/* Mean sparse-softmax cross entropy of code_vec against `target` without gradients
 * (tensorflow_model.py:226-230).  code_vec needs only float alignment: code vectors that are not 16-byte aligned
 * take the fp32 SIMT logits through an aligned copy.  loss_out: device float[1]. */
int c2v_loss(c2v_engine* e, const float* code_vec, const int32_t* target, int32_t B,
             float* loss_out, void* stream);

/* Scores of each example's own name over the whole target vocabulary (NOT IN THE REFERENCE; DESIGN.md §6n): the logits
 * S_b = code_vec_b . TARGET_WORDS_VOCAB^T in the engine's current math mode -- the slab c2v_topk scans, bit for bit --
 * then one pass over each row.  With t_b = S_b[y_b], y_b = target[b], m_b = max_j S_b[j] and
 * lse_b = m_b + log sum_j exp(S_b[j] - m_b):
 *   rank      : 1 + #{j : S_b[j] > t_b} + #{j < y_b : S_b[j] == t_b}, 1-based in tf.nn.top_k's order (value descending,
 *               ties to the lower index): a rank r <= k puts y_b at c2v_topk's idx[b, r - 1]
 *   logp      : t_b - lse_b, the full-softmax log-probability of the target
 *   top1      : the lowest j with S_b[j] == m_b (c2v_topk's idx[b, 0])
 *   top1_logp : m_b - lse_b
 * A row whose logits hold a NaN gets rank 0 and NaN log-probabilities; a target outside [0, target_vocab) rank -1 and
 * NaN log-probabilities.  code_vec: device [B, D] (as c2v_loss); target: device int32 [B]; rank, top1: device int32 [B];
 * logp, top1_logp: device float [B].  No memory beyond the bound workspace.  On a row-sharded target table each engine
 * sees only its rows: the result is its block's, not the model's. */
int c2v_name_scores(c2v_engine* e, const float* code_vec, const int32_t* target, int32_t B,
                    int32_t* rank, float* logp, int32_t* top1, float* top1_logp, void* stream);

/* Forward + backward of the training graph (tensorflow_model.py:197-234 without the Adam
 * update): dropout with keep probability `keep_prob` (config.py:69; 1.0 disables it), full
 * softmax loss, gradients of all five variables written to the bound gradient tensors
 * (overwriting them; embedding rows that received no contribution are exactly 0).
 *   dropout_mask : NULL -> counter-based Philox4x32-10 mask from (seed, step), regenerated in
 *                  the backward pass; or device float [B*C, 3d] of 0/1 supplied by the caller.
 *   loss_out     : device float[1], mean loss over the B examples (dynamic batch, :227).
 * target: device int32 [B]. */
int c2v_train_step(c2v_engine* e, const int32_t* src, const int32_t* path, const int32_t* tgt,
                   const float* mask, const int32_t* target, int32_t B, float keep_prob,
                   uint64_t seed, uint64_t step, const float* dropout_mask, float* loss_out,
                   void* stream);

/* Same with a sampled softmax over {target_b} U sampled[0..S) instead of the full softmax.
 * NOT IN THE REFERENCE (BASELINE config 3; semantics defined in DESIGN.md after
 * tf.nn.sampled_softmax_loss): logq_* are the log expected counts subtracted from the logits,
 * a sampled class equal to a row's target is masked out for that row. */
int c2v_sampled_train_step(c2v_engine* e, const int32_t* src, const int32_t* path,
                           const int32_t* tgt, const float* mask, const int32_t* target,
                           int32_t B, const int32_t* sampled, int32_t S, const float* logq_true,
                           const float* logq_sampled, float keep_prob, uint64_t seed,
                           uint64_t step, const float* dropout_mask, float* loss_out,
                           void* stream);

/* The candidates of one sampled-softmax step, drawn on the device: tf.nn.sampled_softmax_loss's default sampler,
 * tf.random.log_uniform_candidate_sampler(unique=True) (TF's LogUniformSampler with RangeSampler's unique loop), on this
 * library's own random stream.  NOT IN THE REFERENCE (DESIGN.md section 6j).  With Y = target_vocab:
 *   draws    draw i = 0, 1, 2, ... of (seed, step) is r = Philox4x32-10 (common.cuh) at counter (i, 0, step_lo, step_hi)
 *            with key (seed_lo ^ 0x6C6F6775, seed_hi ^ 0x73616D70) -- never the dropout mask's key (seed_lo, seed_hi);
 *            u = ((r.x >> 5) * 2^26 + (r.y >> 6)) * 2^-53, a double in [0, 1); the drawn class is
 *            v = ((int64)floor(exp(u * log1p(Y))) - 1) mod Y, in double.
 *   unique   sampled[0..S) = the first S distinct values in draw order, in the order they first occur; num_tries = the
 *            1-based index of the draw that supplied the S-th distinct value.
 *   counts   in double, rounded to float32 once: p(c) = log((c + 2) / (c + 1)) / log1p(Y); count(c) = S p(c) when
 *            num_tries == S, else -expm1(num_tries * log1p(-p(c))); logq = (float)log(count).  logq_sampled[s] is that of
 *            c = sampled[s], logq_true[b] that of c = target[b] (same num_tries): c2v_sampled_train_step's logq_*.
 * 1 <= S <= min(1024, Y / 2), 1 <= B <= max_batch, else C2V_ERR_INVALID; C2V_ERR_UNSUPPORTED on row-sharded tables
 * (single GPU only).  sampled: device int32 [S]; logq_true: device float [B]; logq_sampled: device float [S]; num_tries:
 * device int64 [1] or NULL.  Asynchronous on `stream`, writes device memory only, allocates nothing (the workspace holds
 * 8 bytes per target class of first-draw stamps).  At most 2^31 draws: a call that reaches that cap without S distinct
 * values fills the missing ids with class 0, reports num_tries = 2^31 and counts itself in the read-only option
 * "sampler_cap_hits" (the read synchronises; it counts the calls of c2v_sample_log_uniform_vocab too). */
int c2v_sample_log_uniform(c2v_engine* e, int32_t S, const int32_t* target, int32_t B, uint64_t seed, uint64_t step,
                           int32_t* sampled, float* logq_true, float* logq_sampled, int64_t* num_tries, void* stream);

/* c2v_sample_log_uniform over an explicit vocabulary of Y classes instead of target_vocab: the same draws, uniqueness,
 * num_tries and log counts, bit for bit, as c2v_sample_log_uniform on an engine whose target_vocab is Y.  Accepted on
 * row-sharded engines, where target_vocab is this rank's block and Y the global vocabulary: every rank that calls it with
 * the same (seed, step) draws the same sampled [S] and logq_sampled [S], and logq_true [B] of its own target ids (global
 * class ids).  NOT IN THE REFERENCE (DESIGN.md section 6j).  2 <= Y, 1 <= S <= min(1024, Y / 2), 1 <= B <= max_batch,
 * else C2V_ERR_INVALID.  The first-draw stamps (8 bytes per class, 2.09 MB at Y = 261,246) are not in the workspace: the
 * first call allocates them (cudaMalloc) and c2v_destroy frees them; a later call with a larger Y synchronises `stream`
 * and allocates again.  A call that reaches the draw cap counts in "sampler_cap_hits" as c2v_sample_log_uniform does. */
int c2v_sample_log_uniform_vocab(c2v_engine* e, int32_t S, int32_t Y, const int32_t* target, int32_t B, uint64_t seed,
                                 uint64_t step, int32_t* sampled, float* logq_true, float* logq_sampled, int64_t* num_tries,
                                 void* stream);

/* tf.compat.v1.train.AdamOptimizer() update of all five variables from the bound gradients
 * (tensorflow_model.py:232): lr_t = lr*sqrt(1-b2^t)/(1-b1^t); m,v decay on EVERY row (TF1's
 * sparse apply is not lazy); theta -= lr_t*m/(sqrt(v)+eps).  t is the 1-based step count. */
int c2v_adam_step(c2v_engine* e, float lr, float beta1, float beta2, float eps, int64_t t,
                  void* stream);

/* Folds the TARGET_WORDS_VOCAB part of that update into the backward pass (tensor-core path, full
 * softmax): once armed, the next target-gradient product dY = P^T.v applies Adam step t to
 * (theta, m, v) of the target table in its epilogue -- bit-identical to c2v_adam_step, but dY is
 * never written (the bound target gradient buffer keeps stale values) and the 401 MB table is not
 * re-read.  The following c2v_adam_step(t) with the same hyper-parameters skips the target table
 * (different ones are an error).  If the step that follows cannot fuse (fp32 path, sampled
 * softmax) the arming is dropped and c2v_adam_step updates the table as usual.  Same semantics as
 * tensorflow_model.py:232; no reference statement of its own. */
int c2v_arm_target_adam(c2v_engine* e, float lr, float beta1, float beta2, float eps, int64_t t);

/* Next-batch hint for "lazy_adam" (one-shot, optional; tf.data's prefetch, path_context_reader.py:150,
 * is what makes the next batch known in the reference too): the index arrays [B, C] of the batch
 * the NEXT train step will run on.  If the current step is armed (c2v_arm_target_adam supplies the
 * step's hyper-parameters) the deferred updates of that batch's embedding rows are applied during
 * the current step's backward pass, on the engine's side stream next to the dY / dW GEMMs,
 * instead of at the head of the next step.  Results are identical with or without the hint; a
 * wrong hint only costs the overlap.  Device pointers must stay valid until the next train step
 * has been issued; the _host variant copies from host memory into the engine's staging area. */
int c2v_hint_next_batch(c2v_engine* e, const int32_t* src, const int32_t* path, const int32_t* tgt,
                        int32_t B);
int c2v_hint_next_batch_host(c2v_engine* e, const int32_t* h_src, const int32_t* h_path,
                             const int32_t* h_tgt, int32_t B, void* stream);

/* ---- Phase-split train step for the fully sharded schedule (BASELINE config 5) -----------------------
 * The target table is row-sharded too: this engine is created with target_vocab = the number of
 * LOCAL rows and max_batch = the GLOBAL batch Bt.  Between the phases the caller moves only small
 * tensors: all-gather of code vectors [Bt, D], all-gather of per-row (max, sum exp) [Bt] and an
 * all-reduce of the true logits [Bt], reduce-scatter of dv [Bt, D] -- never a [*, Y] slab and
 * never a table gradient.
 *   c2v_context_forward : training forward of the local examples (dropout as c2v_train_step) ->
 *                         code_vec [B, D]; activations stay in the workspace for the backward pass.
 *   c2v_target_forward  : S = code_all . Ytab_local^T for all Bt examples; row_max / row_sum [Bt] =
 *                         max and sum exp(. - max) over the local classes; this engine's rows are
 *                         global rows [row_offset, row_offset + target_vocab): true_logit [Bt] =
 *                         S[b, target[b] - row_offset] if that row lives here, else 0
 *                         (target = global class ids of all Bt examples).
 *   c2v_lse_combine     : the ranks' partials maxes / sums [world, Bt] (after all-gather) and the
 *                         all-reduced true logits -> lse [Bt], mean loss (inv_batch = 1/Bt).
 *   c2v_target_backward : S <- (exp(S - lse) - onehot(target - row_offset)) * inv_batch; dv_partial [Bt, D] =
 *                         P . Ytab_local; the bound target gradient (local rows) = P^T . code_all.
 *   c2v_context_backward: rest of the backward pass of the local examples given dv [B, D]
 *                         (after the reduce-scatter): attention, TRANSFORM / ATTENTION gradients,
 *                         scatter-add into the (sharded) embedding gradient tables. */
int c2v_context_forward(c2v_engine* e, const int32_t* src, const int32_t* path, const int32_t* tgt,
                        const float* mask, int32_t B, float keep_prob, uint64_t seed, uint64_t step,
                        const float* dropout_mask, float* code_vec, void* stream);
int c2v_target_forward(c2v_engine* e, const float* code_all, int32_t Bt, const int32_t* target,
                       int32_t row_offset, float* row_max, float* row_sum, float* true_logit,
                       void* stream);
int c2v_lse_combine(c2v_engine* e, const float* maxes, const float* sums, int32_t world, int32_t Bt,
                    const float* true_logit, float inv_batch, float* lse_out, float* loss_out,
                    void* stream);
int c2v_target_backward(c2v_engine* e, const float* code_all, int32_t Bt, const float* lse,
                        const int32_t* target, int32_t row_offset, float inv_batch, float* dv_partial,
                        void* stream);
int c2v_context_backward(c2v_engine* e, const int32_t* src, const int32_t* path, const int32_t* tgt,
                         const float* mask, int32_t B, float keep_prob, uint64_t seed, uint64_t step,
                         const float* dropout_mask, const float* dv, void* stream);

/* ---- Sampled softmax on a row-sharded target table (the fully sharded schedule) -----------------------
 * NOT IN THE REFERENCE (DESIGN.md section 6j).  The same engine as the phase-split step (target_vocab = LOCAL rows
 * [row_offset, row_offset + target_vocab), max_batch = GLOBAL batch Bt = world * B).  The rows move to the examples: every
 * rank draws the same S negatives (c2v_sample_log_uniform_vocab with the global Y and the same seed and step), and a step
 * runs, after c2v_context_forward and an all-gather of the targets into target_all [Bt]:
 *   c2v_sampled_pack_rows   : neg_rows [S, D] row s = Ytab[sampled[s]] and true_rows [Bt, D] row b = Ytab[target_all[b]]
 *                             where this rank holds that row, else zeros.  The caller then all-reduces (sum) neg_rows and
 *                             reduce-scatters (sum) true_rows into its own [B, D] rows; each element has one non-zero
 *                             contributor, so both sums are exact in any order (a -0.0 may become +0.0).
 *   c2v_sampled_target_step : c2v_sampled_train_step's head (fp32 SIMT in every math mode, same operations) on this rank's
 *                             B examples code_vec [B, D] / target [B] (global ids) against the packed rows: logits over
 *                             {true row, S negatives} minus logq_true [B] / logq_sampled [S], accidental hits masked,
 *                             dl = (p - onehot) * inv_batch (pass 1/Bt).  Writes dv [B, D] (c2v_context_backward's input,
 *                             no reduce-scatter needed), loss_partial [1] = (sum_b loss_b) * inv_batch over these B
 *                             examples (fixed order), g_true [B, D] = dl[b,0] * v_b (one product each) and g_neg [S, D] =
 *                             for each s the sums over b of dl[b,1+s] v_b in chunks of 64 examples, added chunk by chunk
 *                             from +0.0f.  No atomics.
 *   c2v_sampled_target_fold : after all-gathers of g_true into g_true_all [Bt, D] (global example order), of g_neg into
 *                             g_neg_all [world, S, D] and of loss_partial into loss_parts [world]: clears the bound target
 *                             gradient block, then stores for every row this rank holds that target_all or sampled
 *                             references, from +0.0f and left to right, g_true_all[b] for each b with target_all[b] == row
 *                             (b order), then for each s with sampled[s] == row (s order) g_neg_all[r][s] for r = 0 ..
 *                             world-1.  loss_out [1] = loss_parts[0] + ... + loss_parts[world-1], left to right from +0.0f,
 *                             the same on every rank.  The target block then takes c2v_adam_step_range (dense TF1 Adam).
 * The whole target side is deterministic by construction.  1 <= S <= 1024, 1 <= B, Bt <= max_batch, 1 <= world <= 8,
 * code_dim <= 1024; code vectors and row buffers 16-byte aligned; else C2V_ERR_INVALID.  The fold needs bound gradients
 * (C2V_ERR_STATE).  Asynchronous on `stream`; dl and the per-example losses live in the workspace. */
int c2v_sampled_pack_rows(c2v_engine* e, const int32_t* sampled, int32_t S, const int32_t* target_all, int32_t Bt,
                          int32_t row_offset, float* neg_rows, float* true_rows, void* stream);
int c2v_sampled_target_step(c2v_engine* e, const float* code_vec, int32_t B, const int32_t* target, const int32_t* sampled,
                            int32_t S, const float* logq_true, const float* logq_sampled, const float* neg_rows,
                            const float* true_rows, float inv_batch, float* dv, float* g_true, float* g_neg,
                            float* loss_partial, void* stream);
int c2v_sampled_target_fold(c2v_engine* e, const float* g_true_all, const float* g_neg_all, int32_t world,
                            const int32_t* target_all, int32_t Bt, const int32_t* sampled, int32_t S, int32_t row_offset,
                            const float* loss_parts, float* loss_out, void* stream);

/* ---- Prediction against a row-sharded target table (the fully sharded schedule) -----------------------
 * The same engine as the phase-split step (target_vocab = LOCAL rows, max_batch = GLOBAL batch Bt).
 * Each rank ranks its own block, the ranks all-gather [Bt, k] candidates, and each rank merges the
 * rows of its own examples; the result is c2v_topk's over the whole target vocabulary: idx equal, val
 * equal for normalize 0 and 1 and equal up to summation order for normalize 2.
 *   c2v_topk_partial : k <= top_k (pass min(top_k, global target vocabulary)).  idx / val [Bt, k] =
 *                      this engine's best k rows for each of the Bt examples, sorted as tf.nn.top_k
 *                      (value descending, ties to the lower id), with GLOBAL ids (local row +
 *                      row_offset) and raw logits, padded with (-inf, INT_MAX) where the block has
 *                      fewer than k rows.  row_max / row_sum [Bt] (both or neither; needed for
 *                      normalize 2) = max and sum exp(. - max) of the example's logits over the
 *                      local rows.  As c2v_topk, lazily updated target rows are brought up to date
 *                      first and 3xTF32 splits the table.  In the tensor-core modes with k <= 16 no
 *                      logit is stored: the logits GEMM's epilogue keeps candidate lists.
 *   c2v_topk_merge   : idx / val [world, Bt, k] (the ranks' c2v_topk_partial results, all-gathered),
 *                      maxes / sums [world, Bt] (their row_max / row_sum; only read for normalize 2)
 *                      -> idx_out / val_out [rows, k] for examples [row0, row0 + rows): the best k of
 *                      the world lists, padding ignored, with c2v_topk's normalize (0, 1, 2; 2 uses
 *                      the global log-sum-exp combined from maxes / sums). */
int c2v_topk_partial(c2v_engine* e, const float* code_all, int32_t Bt, int32_t row_offset, int32_t k,
                     int32_t* idx, float* val, float* row_max, float* row_sum, void* stream);
int c2v_topk_merge(c2v_engine* e, const int32_t* idx, const float* val, const float* maxes,
                   const float* sums, int32_t world, int32_t Bt, int32_t k, int32_t row0, int32_t rows,
                   int32_t normalize, int32_t* idx_out, float* val_out, void* stream);

/* With "lazy_adam" on: replay all deferred updates so that the bound token / path tables (and their
 * Adam slots) hold exactly what the dense optimizer would hold after the steps applied so far.  Call
 * before reading the parameter tensors from outside the engine (export, checkpoint).  No-op otherwise. */
int c2v_sync_tables(c2v_engine* e, void* stream);

/* The same update on one contiguous slice of caller-provided device arrays (count % 4 == 0,
 * 16-byte aligned): the sharded-optimizer path of a data-parallel run, where each rank owns
 * 1/world of the flat parameter buffer (reduce-scatter grads -> this -> all-gather params). */
int c2v_adam_step_range(c2v_engine* e, float* theta, float* grad, float* m, float* v,
                        size_t count, float lr, float beta1, float beta2, float eps, int64_t t,
                        int32_t zero_grad, void* stream);

/* Row-sharded embedding tables over the GPUs of one NVSwitch domain (data-parallel runs).  Global
 * row r of WORDS_VOCAB / PATHS_VOCAB lives on rank (r % world) at local row (r / world); tok[i] /
 * path[i] are device pointers to rank i's shard -- the caller's own allocation for i == rank,
 * CUDA-IPC mappings of the peers' allocations otherwise.  The forward gather then reads peer
 * memory directly and the backward scatter-add issues red.global.add to the owning rank, scaled
 * by grad_scale (1/world for a mean over the global batch): no table gradient is ever
 * all-reduced and each rank updates only its own rows with c2v_adam_step_range.  The caller
 * provides the cross-rank ordering (all scatters done before Adam; all Adams done before the next
 * gather).  world must be 1, 2, 4 or 8.  grads may be NULL (inference). */
typedef struct c2v_table_shards {
  int32_t world;
  int32_t rank;
  float* tok[8];
  float* path[8];
} c2v_table_shards;
int c2v_bind_table_shards(c2v_engine* e, const c2v_table_shards* params, const c2v_table_shards* grads,
                          float grad_scale);

/* Push-based embedding-gradient exchange for row-sharded tables.  Every rank owns an INBOX in peer-visible memory
 * (c2v_ipc_alloc, c2v_scatter_inbox_bytes(dims, world) bytes) with one region per sending rank.  With inboxes bound,
 * the backward pass no longer issues 16-byte red.global.add over NVLink: it sorts its 3 B C gradient rows by owning
 * rank and writes each owner's rows -- (local row id, d floats) -- DENSELY into its region of that owner's inbox with
 * plain coalesced stores; after the caller's cross-rank barrier (the same one that ordered the remote red.adds before)
 * each owner folds its inbox into its own gradient shards with local atomics (c2v_apply_scatter_inbox).  The fold
 * consumes the inbox: a step that pushed nothing (fp32 red.adds straight into the shards) then folds nothing.
 * With option "ordered_exchange" the same inbox carries one fixed-order sum per distinct (owner, table, row) of each
 * sender, token rows then path rows, each list strictly increasing in the local row id, and the fold adds the senders'
 * sums of a row in sender-rank order without atomics and stores the row (see the option).
 * inbox[r] = rank r's inbox as mapped into this process (r == rank: the local allocation). */
size_t c2v_scatter_inbox_bytes(const c2v_dims* dims, int32_t world);
int c2v_bind_scatter_inbox(c2v_engine* e, void* const* inbox, int32_t world, int32_t rank);
int c2v_apply_scatter_inbox(c2v_engine* e, void* stream);

/* cudaMalloc'ed, zero-filled, IPC-shareable device memory for the shards (not tied to an engine;
 * errors are reported through c2v_last_error(NULL)).  handle64 is a 64-byte cudaIpcMemHandle_t. */
int c2v_ipc_alloc(int device, size_t bytes, void** dev_ptr, unsigned char* handle64);
int c2v_ipc_open(int device, const unsigned char* handle64, void** dev_ptr);
int c2v_ipc_close(int device, void* dev_ptr);
int c2v_ipc_free(int device, void* dev_ptr);

/* Register a cudaEvent_t (passed as void*; NULL unregisters) that c2v_train_step records on its
 * stream at a named point, so the caller can start communication early on another stream:
 *   "target_grads_ready" : the TARGET_WORDS_VOCAB gradient is complete (right after dY), while
 *                          the context backward pass is still to run. */
int c2v_set_event(c2v_engine* e, const char* name, void* cuda_event);

/* --- host-buffer entry points: what the backend's train()/evaluate()/predict() call -------- */

/* One `sess.run([optimizer, train_loss])` (tensorflow_model.py:80): copies the batch from host
 * memory (pinned memory makes the copies asynchronous), runs c2v_train_step + c2v_adam_step
 * with the TF defaults given, copies the loss back and synchronises.  h_* are HOST pointers. */
int c2v_train_batch_host(c2v_engine* e, const int32_t* h_src, const int32_t* h_path,
                         const int32_t* h_tgt, const float* h_mask, const int32_t* h_target,
                         int32_t B, float keep_prob, uint64_t seed, int64_t t, float lr,
                         float beta1, float beta2, float eps, float* h_loss, void* stream);

/* The same step WITHOUT waiting for it: the asynchronous half of the batcher that replaces tf.data's prefetch
 * (path_context_reader.py:150).  The five h_* arrays must be page-locked host memory that stays untouched until
 * `upload_done_event` (a cudaEvent_t, may be NULL) has completed: the copies run on an engine-owned copy stream, behind the
 * step that last used the same one of two device staging sets, so the upload of batch t+1 overlaps the kernels of batch t.
 * The step itself (arm target Adam if "fuse_target_adam", train step, Adam step t) is queued on `stream` behind the upload;
 * the loss is copied to h_loss (page-locked, 4 bytes) on `stream` and is valid once `stream` has been synchronised. */
int c2v_train_batch_async(c2v_engine* e, const int32_t* h_src, const int32_t* h_path, const int32_t* h_tgt,
                          const float* h_mask, const int32_t* h_target, int32_t B, float keep_prob,
                          uint64_t seed, int64_t t, float lr, float beta1, float beta2, float eps,
                          float* h_loss, void* upload_done_event, void* stream);

/* One `sess.run([top_words, top_values, ..., code_vectors])` of the test graph
 * (tensorflow_model.py:157-161,331-335).  Outputs are HOST pointers; h_code_vec [B, D] and
 * h_attn [B, C] may be NULL. */
int c2v_predict_batch_host(c2v_engine* e, const int32_t* h_src, const int32_t* h_path,
                           const int32_t* h_tgt, const float* h_mask, int32_t B,
                           int32_t normalize, int32_t* h_topk_idx, float* h_topk_val,
                           float* h_code_vec, float* h_attn, void* stream);

/* Test hook for the tensor-core (wgmma) GEMM building block: C = A . B with tf32 operands.  a_mn / b_mn
 * select the operand layout (0: K contiguous, element (x,k) at p[x*ld+k]; 1: M resp. N
 * contiguous, element (x,k) at p[k*ld+x]); bn is the N tile (192 or 256); with splits > 1,
 * slice s of the K range is written to C + s*M*ldc.  Returns the number of slices (> 0) or an
 * error (< 0).  All pointers are device pointers. */
int c2v_selftest_gemm(c2v_engine* e, int32_t a_mn, int32_t b_mn, int32_t bn, int32_t M, int32_t N,
                      int32_t K, int32_t splits, const float* A, size_t lda, const float* B,
                      size_t ldb, float* C, size_t ldc, void* stream);

/* The same product as 3xTF32 (C2V_MATH_3XTF32): A / A_lo and B / B_lo hold the tf32 high parts and
 * residuals of the fp32 operands (same layout and pitch); c2v_selftest_split produces them
 * (hi = rna_tf32(x), lo = rna_tf32(x - hi); count % 4 == 0, 16-byte aligned device pointers). */
int c2v_selftest_gemm3(c2v_engine* e, int32_t a_mn, int32_t b_mn, int32_t bn, int32_t M, int32_t N,
                       int32_t K, int32_t splits, const float* A, const float* A_lo, size_t lda,
                       const float* B, const float* B_lo, size_t ldb, float* C, size_t ldc,
                       void* stream);
int c2v_selftest_split(c2v_engine* e, const float* x, float* hi, float* lo, size_t count, void* stream);

/* The same product with both operands K contiguous (tf32, no split-K) that also writes B transposed, as the logits GEMM
 * writes the target table's K-major copy for dv: BT[k * ldbt + n] = B[n * ldb + k] for n < N, k < K (columns N .. ldbt-1
 * are not written).  K % 4 == 0, ldbt >= N and ldbt % 4 == 0, BT 16-byte aligned. */
int c2v_selftest_gemm_bt(c2v_engine* e, int32_t M, int32_t N, int32_t K, const float* A, size_t lda, const float* B,
                         size_t ldb, float* C, size_t ldc, float* BT, size_t ldbt, void* stream);

/* Test hook for the K-major copies the engine makes of its MN-major GEMM operands: xT[c, r] = x[r, c] for a row-major
 * x [rows, cols] (pitch cols) into xT [cols, ldT] (ldT >= rows; columns rows .. ldT-1 are not written).  With xT_lo
 * non-NULL, xT / xT_lo receive the transposed 3xTF32 split of x instead.  Device pointers. */
int c2v_selftest_transpose(c2v_engine* e, const float* x, int32_t rows, int32_t cols, float* xT, float* xT_lo, size_t ldT,
                           void* stream);

/* Test hook: where the bound workspace holds the K-major copy of the target table that the dv GEMM reads, Ytab^T
 * [code_dim, *ld] (columns target_vocab .. *ld-1 are padding): lo = 0 the table itself (tf32) or its transposed high parts
 * (3xTF32), lo = 1 the transposed residuals (3xTF32).  *offset is in bytes from the workspace base. */
int c2v_selftest_target_t(const c2v_engine* e, int32_t lo, size_t* offset, size_t* ld);

/* Test hook for option "deterministic": the sort + chunked reduce of a train step's embedding-gradient scatter, on
 * `count` caller-given contributions instead of dX' (no dropout, no scaling): row rows[i] of table table_id (0 = token
 * table [T, d], 1 = path table [P, d]; d = embed_dim) receives vals[i, 0:d], summed in the order the option documents,
 * and is stored into out (the table, zero on entry: unreferenced rows are not written).  count <= 3 * max_batch *
 * max_contexts; rows must be in range; vals and out are 16-byte aligned device pointers. */
int c2v_selftest_row_sum(c2v_engine* e, int32_t table_id, const int32_t* rows, const float* vals, int32_t count,
                         float* out, void* stream);

/* Test hook for option "ordered_exchange": the sender's half of the exchange on caller-given contributions instead of
 * dX' (no dropout, no scaling).  GLOBAL token row tok_rows[i] receives tok_vals[i, 0:d] and global path row path_rows[i]
 * receives path_vals[i, 0:d]; per distinct row the contributions are summed in list order as "deterministic" documents
 * and pushed into the owners' inboxes.  The caller then barriers and calls c2v_apply_scatter_inbox on every rank.  Needs
 * the option set, shards bound over more than one rank and an inbox bound; n_tok + n_path <= 3 * max_batch *
 * max_contexts; rows in range; 16-byte aligned device pointers (a list of length 0 may be NULL). */
int c2v_selftest_exchange_push(c2v_engine* e, const int32_t* tok_rows, const float* tok_vals, int32_t n_tok,
                               const int32_t* path_rows, const float* path_vals, int32_t n_path, void* stream);

/* Introspection for tests and bench: number of kernels the engine has launched so far. */
int64_t c2v_launch_count(const c2v_engine* e);

/* Per-phase device timing (option "profile" = 1): CUDA events bracket every phase of a pass on
 * the launching stream.  c2v_phase_stats synchronises, folds the pending events into the
 * running totals and returns them (reset != 0 clears the totals afterwards). */
int c2v_phase_count(void);
const char* c2v_phase_name(int phase);
int c2v_phase_stats(c2v_engine* e, int phase, double* total_ms, int64_t* count, int reset);

/* ---- Device reader (DESIGN.md §6d) ------------------------------------------------------------------------------
 * Turns `.c2v` training text in device memory into the rows of a training shuffle pool held on the device, and draws
 * batches from that pool into caller buffers: the host reader's train path (path_context_reader.py
 * _iterate_batches_native: native/batcher.cpp c2v_parse_chunk in train mode, _RowPool.commit, _RowPool.take) with every
 * row, every pool move and every batch identical to the host's for the same draws.  A reader handle is independent of
 * any engine handle.  Failures return a negative c2v_status with the message in c2v_last_error(NULL) (of the calling
 * thread).  Calls on one handle run on one caller stream (or the caller orders them); one host thread at a time. */
typedef struct c2v_reader c2v_reader;

/* One vocabulary as native/batcher.cpp holds it (c2v_vocab_export), copied to the device by the caller and kept alive
 * until c2v_reader_destroy: slots [mask + 1] of 24 bytes {uint64 h (FNV-1a 64 of the word, 0 = empty), int64 off,
 * int32 len, int32 idx}, probed linearly from h & mask; bytes: the words, concatenated. */
typedef struct c2v_reader_vocab {
  const void* slots;
  const char* bytes;
  uint64_t mask;
  int32_t oov;     /* index of an unknown word (and of an empty target) */
  int32_t pad;     /* index of an absent context part                     */
} c2v_reader_vocab;

/* A reader for rows of max_contexts contexts on `device`, with an empty pool.  The handle allocates its own device
 * buffers (pool, per-chunk scratch), growing them as chunks and draws need; c2v_reader_device_bytes reports them. */
int c2v_reader_create(int32_t max_contexts, const c2v_reader_vocab* token, const c2v_reader_vocab* path,
                      const c2v_reader_vocab* target, int device, c2v_reader** out);
void c2v_reader_destroy(c2v_reader* r);      /* synchronises the device, then frees the handle's buffers */

/* Parses the complete lines of text[0, nbytes) (device memory; the last line may lack its newline) as c2v_parse_chunk
 * does in train mode -- trailing '\r' stripped, blank lines skipped, exactly max_contexts + 1 space-separated fields, at
 * most 3 comma-separated parts per context, the row filter "any index != PAD and target > OOV" -- and appends the kept
 * rows behind the pool's live end in the host pool's order (_RowPool.commit: the j-th dropped row below the kept count
 * takes the j-th kept row beyond it).  Synchronises `stream` and sets *kept to the rows added.  A malformed chunk leaves
 * the pool unusable and returns C2V_ERR_INVALID with *bad_line = the lowest malformed line's number (0-based, blank
 * lines counted) and *bad_kind = 1 (field count) or 2 (a context with more than 3 parts), or *bad_kind = 3 when the
 * chunk has more lines than nbytes / (max_contexts + 1) + 1, which no well-formed chunk has. */
int c2v_reader_parse_chunk(c2v_reader* r, const char* text, int64_t nbytes, int64_t* kept, int64_t* bad_line,
                           int32_t* bad_kind, void* stream);

/* One draw of b rows from the pool's n live rows (_RowPool.take / c2v_pool_take): pick[0, b) are b distinct row
 * indices in [0, n) (host memory; page-locked keeps the copy asynchronous; unchanged until the draw has run).  Rows
 * pick[lo, hi) are written to src / path / tgt / mask [hi - lo, max_contexts] and target [hi - lo] (device memory; may
 * be NULL when lo == hi), then the holes the picks leave below n - b are filled with the tail rows that were not
 * picked, both in ascending order.  A rank of a multi-GPU run passes its slice [lo, hi) of the global batch and draws
 * the whole pick, so every rank's pool stays the same.  Asynchronous on `stream`. */
int c2v_reader_draw(c2v_reader* r, const int64_t* pick, int32_t b, int32_t lo, int32_t hi, int32_t* src, int32_t* path,
                    int32_t* tgt, float* mask, int32_t* target, void* stream);

/* Rows in the pool once the queued calls have run (-1 for a NULL handle); device memory the handle holds (pool, scratch,
 * and the evaluation queue and tables). */
int64_t c2v_reader_live_rows(const c2v_reader* r);
size_t c2v_reader_device_bytes(const c2v_reader* r);

/* A chunk read sharded across W ranks (device_reader.py, DESIGN.md §6d).  The chunk's text is cut at line starts into W
 * shares in rank order; each rank parses its own share into a *stage*, a peer-visible device allocation (c2v_ipc_alloc)
 * of c2v_reader_stage_bytes(max_contexts, rows) bytes, and every rank then commits all W stages, its own and its peers'
 * (opened through CUDA IPC), into its pool.  The pool that results is the one c2v_reader_parse_chunk builds from the
 * whole chunk, and the chunk's error is decided from the W statuses: with R = the sum of their records and
 * cap = chunk_bytes / (max_contexts + 1) + 1, kind 3 if R > cap, otherwise the lowest malformed line over the shares
 * (each share's bad_line plus the newlines of the shares before it) with its share's kind.
 * A stage holds this status in its first 256 bytes, then the rows and keep flags of up to `rows` records. */
typedef struct c2v_reader_share_status {
  int64_t rows;        /* the stage's row capacity                                                              */
  int64_t records;     /* records (non-blank lines) of the share                                                 */
  int64_t kept;        /* records that pass the training filter (0 when the share is malformed or overflows)     */
  int64_t newlines;    /* '\n' bytes of the share                                                                 */
  int64_t bad_line;    /* the share's lowest malformed line, counted from the share's first byte, or -1          */
  int32_t bad_kind;    /* 1 (field count), 2 (a context with more than 3 parts) or 0                             */
  int32_t overflow;    /* records > rows: the share holds a malformed line, or more records than the chunk allows */
} c2v_reader_share_status;

/* Bytes of a stage of `rows` rows (0 for max_contexts < 1 or rows < 1). */
size_t c2v_reader_stage_bytes(int32_t max_contexts, int64_t rows);

/* Parses the share text[0, nbytes) (device memory, whole lines) of a chunk of chunk_bytes bytes into `stage` (device
 * memory of c2v_reader_stage_bytes(max_contexts, stage_rows) bytes) with c2v_reader_parse_chunk's rules, writes the
 * share's status into the stage and *status, and synchronises `stream`.  A share with more records than stage_rows
 * rows (a share of n bytes needs at most n / (max_contexts + 1) + 1) is malformed; its lowest malformed line is then
 * found in the handle's own pool room, unless it has more records than the whole chunk allows.  A malformed share
 * returns C2V_OK: the chunk's error is decided from every share's status.  The pool is not touched otherwise. */
int c2v_reader_parse_share(c2v_reader* r, const char* text, int64_t nbytes, int64_t chunk_bytes, void* stage,
                           int64_t stage_rows, c2v_reader_share_status* status, void* stream);

/* Appends the chunk of n_shares parsed shares (1 <= n_shares <= 64) to the pool: stages[i] (this device's memory or a
 * peer's opened through CUDA IPC; may be NULL when records[i] == 0) holds share i's records[i] records, shares in rank
 * order.  The rows and keep flags of every stage are copied behind the live end (kernel assemble_shares_kernel) and the
 * chunk's records are committed as c2v_reader_parse_chunk commits them.  Call it only for a chunk whose shares all
 * parsed clean and whose record total is within the chunk's cap.  Synchronises `stream` (so no stage is read once it
 * returns) and sets *kept to the rows added. */
int c2v_reader_commit_shares(c2v_reader* r, const void* const* stages, const int64_t* records, int32_t n_shares,
                             int64_t* kept, void* stream);

/* ---- Evaluation on the device (DESIGN.md §6e) ----------------------------------------------------------------------
 * A reader handle also reads `.c2v` test files: c2v_reader_eval_append parses a chunk in evaluate mode and appends the
 * kept rows to an evaluation queue in file order, c2v_reader_eval_take hands out the next rows with their names, and
 * c2v_reader_eval_score scores the engine's top-k ids of a batch against the names.  This is the host reader's evaluate
 * path (path_context_reader.py _iterate_batches_native with c2v_parse_chunk mode 1) and the host metrics
 * (common.get_first_match_word_from_top_predictions, SubtokensEvaluationMetric.update_batch) row for row.  The evaluation
 * queue does not touch the training pool: a handle can serve both, but a reader of one kind is the usual use. */

/* Uploads the per-target-word tables the evaluation needs, computed on the host from the target vocabulary (host
 * memory; copied before the call returns): word i's bytes are words[word_off[i], word_off[i + 1]), its normalize_word
 * bytes norm[norm_off[i], norm_off[i + 1]), and legal[i] != 0 when legal_method_names_checker accepts it.  n_words must
 * cover the target vocabulary, its OOV word included: an empty name stands for that word.  Replaces earlier tables. */
int c2v_reader_eval_tables(c2v_reader* r, int32_t n_words, const char* words, const int64_t* word_off, const char* norm,
                           const int64_t* norm_off, const uint8_t* legal, void* stream);

/* Parses the complete lines of text[0, nbytes) (device memory) with c2v_reader_parse_chunk's rules but the evaluate
 * filter -- a record is kept when any of its contexts is valid, whatever its target -- and appends the kept rows, in
 * file order, to the evaluation queue.  Each row keeps its name: field 0's bytes (commas included), or the target OOV
 * word's when field 0 is empty.  Needs the tables (C2V_ERR_STATE otherwise).  Synchronises `stream`; *appended = the rows
 * added, *name_bytes = the name bytes the queue holds now (a bound on the names of any take before the next append).
 * Errors as c2v_reader_parse_chunk, with nothing appended. */
int c2v_reader_eval_append(c2v_reader* r, const char* text, int64_t nbytes, int64_t* appended, int64_t* name_bytes,
                           int64_t* bad_line, int32_t* bad_kind, void* stream);

/* Moves the next b queued rows (1 <= b <= c2v_reader_eval_queued) into src / path / tgt / mask [b, max_contexts] and
 * target [b] (device memory), and their names into names (device memory of names_cap bytes, at least the *name_bytes
 * the last append reported) with row j's name at names[name_off[j], name_off[j + 1]) (name_off: device, [b + 1]).
 * Asynchronous on `stream`. */
int c2v_reader_eval_take(c2v_reader* r, int32_t b, int32_t* src, int32_t* path, int32_t* tgt, float* mask,
                         int32_t* target, int64_t* name_off, char* names, int64_t names_cap, void* stream);

/* Rows queued and not yet taken (-1 for a NULL handle). */
int64_t c2v_reader_eval_queued(const c2v_reader* r);

/* Scores n rows: ids [n, k] (device; the engine's top-k word ids, best first) against the names
 * names[name_off[j], name_off[j + 1]) (device, as c2v_reader_eval_take writes them).  Per row (device outputs [n]):
 * rank[j] = the rank of the first word whose normalize_word equals the name's among the legal words of the top-k (not
 * among all k), or -1; first[j] = the id of the first legal word, or -1; flags[j] = 1 when the name has a byte >= 0x80
 * (the host scores it: normalize_word and the UTF-8 decoding are Unicode), 2 when no word of the top-k is legal (the host
 * raises, as the host metric does), else 0.  acc (device int64 [k + 4], zeroed here) sums the unflagged rows: a histogram
 * of their ranks over [0, k), then their number, and the subtoken true positives, false positives and false negatives of
 * the first legal word against the name ('|'-separated, empty subtokens included, multiset counts).  Integer sums: the
 * result does not depend on the order rows are added.  Only reads the handle's tables, so it may run on another host
 * thread than append / take.  Asynchronous on `stream`. */
int c2v_reader_eval_score(const c2v_reader* r, const int32_t* ids, int32_t n, int32_t k, const int64_t* name_off,
                          const char* names, int32_t* rank, int32_t* first, int32_t* flags, int64_t* acc, void* stream);

/* Checks the names of the last `rows` queued rows (0 <= rows <= c2v_reader_eval_queued; after an append, the rows it
 * added) against Python's strict UTF-8 decoder: no overlong forms, no surrogates, nothing above U+10FFFF.  *name_len
 * (host) = -1 when every name is valid; otherwise the length of the first invalid name in queue order, whose first
 * min(len, name_cap) bytes go to name (host), so the caller can raise the decoder's own error from them.  Synchronises. */
int c2v_reader_eval_check_utf8(c2v_reader* r, int64_t rows, char* name, int64_t name_cap, int64_t* name_len, void* stream);

/* The target-word bytes of the tables (device memory of the handle, valid until the tables are replaced or the handle
 * destroyed): word i is (*words)[(*word_off)[i], (*word_off)[i + 1]) for i < *n_words.  C2V_ERR_STATE before the tables. */
int c2v_reader_eval_words(const c2v_reader* r, const char** words, const int64_t** word_off, int32_t* n_words);

/* ---- Text of float32 matrices (DESIGN.md §6f) -----------------------------------------------------------------------
 * The lines of `<test file>.vectors` (model_base._write_code_vectors) and of word2vec files (common.save_word2vec_file),
 * formatted on the device.  Every value is written as numpy's str(np.float32(x)) writes it: "nan", "inf", "-inf",
 * "0.0", "-0.0"; positional ("0.5", "999999.0", "0.000100000005") for 1e-4 <= |x| < 1e6, compared exactly; otherwise
 * scientific ("1e+07", "1.5e+08", "1.1754944e-38"); digits of Dragon4 in numpy's "unique" mode.  No engine handle is
 * needed; failures return a negative c2v_status with the message in c2v_last_error(NULL). */

/* Bytes one value's text and the separator after it take at most (a value is at most 15 bytes long). */
#define C2V_TEXT_VALUE_BYTES 16

/* Formats rows [0, rows) of the row-major float32 matrix x (device; row r at x + r * ld, cols values) as lines: row r's
 * prefix bytes prefix[prefix_off[r], prefix_off[r + 1]) (device; both NULL for no prefix), then its values joined by
 * single spaces, then '\n'.  stage (device, stage_bytes >= rows * cols * C2V_TEXT_VALUE_BYTES) is scratch.  row_end
 * (device, [rows]) receives each line's end offset in out, lines back to back from out[0]; *rows_done (device) = the
 * lines that end within out_cap bytes, which are written to out (device); the others are left for the next call.
 * Asynchronous on `stream`. */
int c2v_text_format_rows(const float* x, int64_t rows, int32_t cols, int64_t ld, const char* prefix,
                         const int64_t* prefix_off, void* stage, size_t stage_bytes, char* out, int64_t out_cap,
                         int64_t* row_end, int64_t* rows_done, void* stream);

/* Test hook: formats x[0, n) (host) on the CPU with the function the device runs.  Value i's text goes to
 * out[i * C2V_TEXT_VALUE_BYTES, ...) followed by NUL bytes up to the next value, and its length to len[i] (host). */
int c2v_selftest_format_floats(const float* x, int64_t n, char* out, int32_t* len);

/* ---- CRC-32C of device memory (DESIGN.md §6k) ------------------------------------------------------------------------
 * The checksum of a TensorFlow tensor bundle entry (tf_bundle.py): CRC-32C, reflected polynomial 0x82F63B78, init and
 * xorout 0xFFFFFFFF ("123456789" -> 0xE3069283).  No engine handle is needed; any alignment is accepted; failures return
 * a negative c2v_status with the message in c2v_last_error(NULL).  Asynchronous on `stream`. */

/* crc_out[r] (device, [rows]) = the CRC-32C of the row_bytes bytes at base + r * row_stride (device), r in [0, rows).
 * A row of no bytes has CRC 0. */
int c2v_crc32c_rows(const void* base, int64_t rows, int64_t row_bytes, int64_t row_stride, uint32_t* crc_out,
                    void* stream);

/* *out (device) = the CRC-32C of the concatenation of n segments of seg_bytes bytes each, from their CRCs crcs[0, n)
 * (device): zlib's crc32_combine as a tree reduction.  n = 0 gives 0. */
int c2v_crc32c_combine(const uint32_t* crcs, int64_t n, int64_t seg_bytes, uint32_t* out, void* stream);

/* ---- The Keras output kernel's transpose (DESIGN.md §6l) ----------------------------------------------------------------
 * Keras stores the output layer's kernel as [D, Y]; the engine holds it as [Y, ld].  These move a chunk of k file rows
 * between the two layouts as exact bit copies (NaN payloads and -0.0 included).  Any k >= 0, Y >= 0, col0 >= 0 with
 * ld >= col0 + k; src and dst are device pointers aligned to 4 bytes.  No engine handle is needed; failures return a
 * negative c2v_status with the message in c2v_last_error(NULL).  Asynchronous on `stream`. */

/* dst[y * ld + col0 + i] = src[i * Y + y] for i < k, y < Y: k file rows into columns [col0, col0 + k) of dst. */
int c2v_rows_to_cols(const float* src, int64_t k, int64_t Y, float* dst, int64_t ld, int64_t col0, void* stream);

/* dst[i * Y + y] = src[y * ld + col0 + i] for i < k, y < Y: columns [col0, col0 + k) of src into k file rows. */
int c2v_cols_to_rows(const float* src, int64_t ld, int64_t col0, int64_t k, int64_t Y, float* dst, void* stream);

/* ---- Preprocessing on the device (DESIGN.md §6g) ----------------------------------------------------------------------
 * Raw extractor output (`target ctx ctx ...` lines) in device memory -> what preprocess.py's count_histograms and
 * process_file write, byte for byte (device_preprocess.py).  A chunk is whole lines of a file under universal newlines:
 * it ends after '\n', after a '\r' that the file does not follow with '\n', or at the end of the file.  Lines are split
 * on ' ' into fields (field 0 the target, the others contexts, empty ones included) and contexts on ','.  A handle is
 * independent of any engine or reader handle.  Failures return a negative c2v_status with the message in
 * c2v_last_error(NULL).  Calls on one handle run on one caller stream, one host thread at a time; each call below that
 * reports a status synchronises the stream. */
typedef struct c2v_prep c2v_prep;

typedef struct c2v_prep_status {
  int64_t lines;       /* lines of the chunk, blank ones included                                                   */
  int64_t bad_utf8;    /* offset in the chunk of the first byte Python's strict UTF-8 decoder rejects, or -1; the
                          chunk is not processed further when it is set                                             */
  int64_t bad_line;    /* classify: the first line (0-based in the chunk) with more than max_contexts contexts and a
                          context of fewer than 3 parts (process_file raises IndexError there), or -1             */
  int64_t long_lines;  /* classify: lines with more than max_contexts contexts                                     */
  int64_t seen, kept, written, empty, longest;   /* classify: process_file's statistics over the chunk's lines      */
  int64_t keys;        /* count: distinct keys in the histogram table (all three kinds)                             */
  int64_t slots;       /* count: slots of the table                                                                 */
  int64_t rehashes;    /* count: times the table was doubled with keys in it                                        */
} c2v_prep_status;

int c2v_prep_create(int device, c2v_prep** out);
void c2v_prep_destroy(c2v_prep* h);          /* synchronises the device, then frees the handle's buffers */
size_t c2v_prep_device_bytes(const c2v_prep* h);     /* device memory the handle holds (table, arena, scratch) */

/* count_histograms over the chunk text[0, nbytes) (device memory, nbytes < 2^31) that starts at byte file_offset of
 * the file: per line tokens[p0], paths[p1], tokens[p2] of every context of 3 parts or more (later parts ignored),
 * tokens[p0] and, with a second part, paths[p1] of the others, and targets[field 0].  Counts add up across calls; each
 * key keeps the file offset of its first occurrence.  The table doubles (rehash) before a chunk whose inserts could
 * take it past half full; key bytes are copied to an arena, so the text may be reused once this returns. */
int c2v_prep_count_chunk(c2v_prep* h, const char* text, int64_t nbytes, int64_t file_offset, c2v_prep_status* st,
                         void* stream);

/* The histogram of kind 0 (tokens), 1 (paths) or 2 (targets) as write_histogram writes a Counter: `word count\n` per
 * key, keys in the order of their first occurrence.  *text (device memory of the handle, valid until the next call on
 * it) and *nbytes receive the text. */
int c2v_prep_histogram(c2v_prep* h, int32_t kind, const char** text, int64_t* nbytes, void* stream);

/* The down-sampling decisions of process_file for the chunk text[0, nbytes) (device memory, kept unchanged until
 * c2v_prep_assemble has run): every context's bytes, and for each line of more than max_contexts contexts its full
 * (all three parts in the vocabularies: token and path are membership tables built as c2v_reader_vocab, a word is in
 * when its index is not oov) and partial contexts in file order.  st gets the chunk's statistics. */
int c2v_prep_classify_chunk(c2v_prep* h, const char* text, int64_t nbytes, int32_t max_contexts,
                            const c2v_reader_vocab* token, const c2v_reader_vocab* path, c2v_prep_status* st,
                            void* stream);

/* Per line of more than max_contexts contexts of the classified chunk, in file order (host outputs [st.long_lines]):
 * its line in the chunk, its full and its partial context counts. */
int c2v_prep_long_lines(c2v_prep* h, int64_t* line, int32_t* n_full, int32_t* n_partial, void* stream);

/* The lines process_file writes for the classified chunk: long line r (in c2v_prep_long_lines order) takes
 * picks[pick_off[r], pick_off[r + 1]) (host memory): with n_full > max_contexts, max_contexts indices into its full
 * contexts (rng.sample(range(n_full), max_contexts)); with n_full + n_partial > max_contexts, max_contexts - n_full
 * indices into its partial contexts after all the full ones; otherwise none (its full, then its partial contexts).
 * Output contexts keep the pick order; a line is `target ctx ... ctx` + the padding spaces up to max_contexts contexts
 * + '\n', and lines left with no context are skipped.  *text (device memory of the handle, valid until the next call)
 * and *nbytes receive the chunk's lines; the copy is ordered on `stream`.  C2V_ERR_STATE when bad_line was set. */
int c2v_prep_assemble(c2v_prep* h, const int32_t* picks, const int64_t* pick_off, const char** text, int64_t* nbytes,
                      void* stream);

/* ---- Nearest neighbours (DESIGN.md §6h) ------------------------------------------------------------------------------
 * Cosine search over the rows of a float32 table T [rows, dim] in device memory: gensim 4's KeyedVectors.most_similar on
 * the embedding tables, and the nearest methods of a corpus by code vector (similarity.py).  With norm_i = ||T_i||, row
 * i scores s_i = (T_i . q) / norm_i against a query q; a row of zero norm (or with a NaN) scores NaN and is never
 * returned.  Results are ordered as tf.nn.top_k orders them: value descending, exact ties to the lower row.  A handle is
 * independent of any engine handle; failures return a negative c2v_status with the message in c2v_last_error(NULL).
 * Calls on one handle run on one caller stream, one host thread at a time. */
typedef struct c2v_knn c2v_knn;

int c2v_knn_create(int device, c2v_knn** out);
void c2v_knn_destroy(c2v_knn* h);          /* synchronises the device, then frees the handle's buffers */

/* The most device memory the handle has held at once (norms, table copies, one query block's buffers). */
size_t c2v_knn_device_bytes(const c2v_knn* h);

/* Binds T (row r at table + r * ld; 1 <= dim <= ld, rows < 2^31) with the arithmetic of the searches (c2v_math_mode):
 * computes the row norms (in double) and, in 3xTF32, the tf32 split of the table; a table without a 16-byte row pitch
 * is also copied with one.  T must stay allocated while bound; once its contents change, bind it again (the norms and
 * copies describe the contents at this call).  Asynchronous on `stream`. */
int c2v_knn_bind_table(c2v_knn* h, const float* table, int64_t rows, int32_t dim, int64_t ld, int32_t math, void* stream);

/* gensim's query vectors (KeyedVectors.get_mean_vector with pre- and post-normalisation): query j is the sum over
 * e in [offsets[j], offsets[j + 1]) of weights[e] * T[word_ids[e]] / norm, computed in double and scaled to unit length
 * (a zero sum stays zero), written as float to q_out [nq, dim] (pitch dim).  word_ids (in [0, rows)), weights
 * (+1 positive, -1 negative), offsets [nq + 1] and q_out are device memory.  Asynchronous on `stream`. */
int c2v_knn_queries(c2v_knn* h, const int32_t* word_ids, const float* weights, const int64_t* offsets, int32_t nq, float* q_out,
                    void* stream);

/* For each query j of q [nq, dim] (pitch ldq >= dim, device): the k + max_exclude best rows, then without the ids
 * exclude[exclude_off[j], exclude_off[j + 1]) (device; NULL when max_exclude = 0; a list has at most max_exclude
 * entries), the first k of the rest -> idx / val [nq, k] (device), padded with (INT_MAX, -inf) where fewer rows remain.
 * That is gensim's exclusion of the query words from the top topn + len(words).  k + max_exclude <= 64.
 * Routes: tf32 / 3xTF32 with k + max_exclude <= 16, the wgmma GEMM whose epilogue scales each column by 1 / norm and
 * keeps candidate lists, merged per query; otherwise (fp32, or more candidates) the fp32 SIMT GEMM into a score slab
 * and the top-k kernels.  Queries go in blocks whose candidate lists or slab take at most 512 MB and that hold at most
 * 65536 queries, so the memory held does not grow with nq.  Asynchronous on `stream`. */
int c2v_knn_search(c2v_knn* h, const float* q, int32_t nq, int64_t ldq, int32_t k, const int32_t* exclude,
                   const int64_t* exclude_off, int32_t max_exclude, int32_t* idx, float* val, void* stream);

/* Device time of the searches since the last call, split into the GEMM (with its candidate epilogue) and the selection
 * (merge or slab top-k, exclusion), in ms; synchronises.  on != 0 times the searches that follow (CUDA events around
 * each query block), 0 stops. */
int c2v_knn_profile(c2v_knn* h, int32_t on, double* gemm_ms, double* select_ms);

/* ---- Device predict (DESIGN.md §6i) ---------------------------------------------------------------------------------
 * `--predict` over extractor output in device memory (device_predict.py): the model input rows of its methods and the
 * text __main__.print_predictions writes for them, byte for byte.  The input must be ASCII.  A handle is independent of
 * any engine handle and reads the vocabularies' device tables (c2v_reader_vocab, as c2v_reader_create) while it lives;
 * failures return a negative c2v_status with the message in c2v_last_error(NULL).  One caller stream, one host thread. */
typedef struct c2v_pred c2v_pred;

int c2v_pred_create(int device, int32_t max_contexts, const c2v_reader_vocab* tok, const c2v_reader_vocab* path,
                    c2v_pred** out);
void c2v_pred_destroy(c2v_pred* h);        /* synchronises the device, then frees the handle's buffers */

/* The most device memory the handle has held at once. */
size_t c2v_pred_device_bytes(const c2v_pred* h);

/* The predicted-name text of every target word: word i's bytes are repr[repr_off[i], repr_off[i + 1]) (host arrays,
 * copied; str(word.split("|")) on the host).  Ids outside [0, n_words) and `oov` are not printed. */
int c2v_pred_set_targets(c2v_pred* h, int32_t n_words, const char* repr, const int64_t* repr_off, int32_t oov, void* stream);

/* The input goes through the handle in chunks of whole lines (each ending at a '\n', or at the end of the input), in
 * three passes: every chunk with C2V_PRED_KEYS, then c2v_pred_seal_keys, every chunk with C2V_PRED_PATHS, then, for
 * predicting, each chunk with C2V_PRED_SCAN followed by c2v_pred_rows / c2v_pred_format on its methods.
 * c2v_pred_reset_keys starts the first pass over.  Only the current chunk is held on the device.
 *
 * A chunk's lines end at '\n' and, with universal_newlines != 0 (a file opened in text mode), also at a '\r' not
 * followed by '\n'.  Each line is rstripped; it is a method when its first ' '-separated field is not empty, and its first
 * max_contexts non-empty fields after that are its contexts, each of which must have exactly two commas.  Every context's
 * path has a key: the path itself when it is -?[0-9]+, else the decimal of its Java String.hashCode.  Per key, the handle
 * keeps the path text of the last context in the input that has it (the largest file_offset + position).
 *   C2V_PRED_SCAN  : index and scan the chunk's lines (c2v_pred_line_info, c2v_pred_rows read them)
 *   C2V_PRED_KEYS  : the same, and record every kept context's key (file_offset: the chunk's offset in the input)
 *   C2V_PRED_PATHS : copy the path texts the table names that lie in this chunk (no line index)
 * Returns the chunk's number of lines (0 for C2V_PRED_PATHS); synchronises. */
#define C2V_PRED_SCAN 0
#define C2V_PRED_KEYS 1
#define C2V_PRED_PATHS 2
int c2v_pred_reset_keys(c2v_pred* h, void* stream);
int c2v_pred_chunk(c2v_pred* h, const char* text, int64_t nbytes, int64_t file_offset, int32_t universal_newlines,
                   int32_t mode, int64_t* n_lines, void* stream);
/* After the last C2V_PRED_KEYS chunk: sizes the arena of path texts.  Synchronises. */
int c2v_pred_seal_keys(c2v_pred* h, void* stream);

/* Per line of the current chunk (host arrays [n_lines]): the rstripped line [lo, hi) in the chunk, its kind (0 skipped,
 * 1 method, 2 a kept context without exactly three comma-separated parts, 3 a path whose key the table cannot hold: a
 * numeric path that is not the canonical decimal of an int32, such as "007", or a path of 1 MB or more) and its number of
 * kept contexts (up to the first bad one).  Synchronous. */
int c2v_pred_line_info(c2v_pred* h, int64_t* lo, int64_t* hi, int32_t* kind, int32_t* kept);

/* The model input of the n methods on lines lines[0, n) of the current chunk (host; all of kind 1): src / path / tgt [n, max_contexts] int32
 * and mask [n, max_contexts] float32 (device), as PathContextReader._map_raw_dataset_row_to_input_tensors builds them
 * from __main__.prepare_extracted_lines' line.  The rows' contexts are kept for the next c2v_pred_format.  Synchronises. */
int c2v_pred_rows(c2v_pred* h, const int64_t* lines, int32_t n, int32_t* src, int32_t* path, int32_t* tgt, float* mask,
                  void* stream);

/* The text of the n rows of the last c2v_pred_rows: for each, "Original name:", the predictions idx / val [n, k], the
 * "Attention:" lines from attn [n, max_contexts] and, when code_vec [n, code_dim] is not NULL, "Code vector:" and its
 * line (all device), once the C2V_PRED_PATHS pass is done.  Written back to back at out (device) when they fit
 * out_cap; *total (host) gets their length either way, and *bad_row (host) the lowest row whose distinct contexts have
 * NaN and non-NaN attention (a value >= n if none; nothing is written then).  Asynchronous: *total and *bad_row are
 * valid once `stream` has completed, so they should be page-locked. */
int c2v_pred_format(c2v_pred* h, int32_t n, const int32_t* idx, const float* val, int32_t k, const float* attn,
                    const float* code_vec, int32_t code_dim, char* out, int64_t out_cap, int64_t* total, int32_t* bad_row,
                    void* stream);

/* Test hook, on the CPU: Python's '%f' % float(x[i]) as the device formats it, into out[i * C2V_FIXED_BYTES, ...)
 * padded with NUL bytes, and its length to len[i] (host). */
#define C2V_FIXED_BYTES 48
int c2v_selftest_format_fixed(const float* x, int64_t n, char* out, int32_t* len);

/* ---- Corpus text (DESIGN.md §6o) --------------------------------------------------------------------------------------
 * The lines of `<corpus>.name_scores` (name_scores.format_line) and `<corpus>.nearest` (similarity.format_nearest_line)
 * formatted on the device, byte for byte.  Names and words are bytes, copied as they are; floats are Python's '%f' of
 * the float32 ("nan", "inf", "-inf", "-0.000000" as the host prints them); integers are '%d'.  Lines go back to back
 * from out[0] (device) when all of them fit out_cap bytes, and *total (host, page-locked: written asynchronously, valid
 * once `stream` has completed) gets their length either way.  scratch (device) holds at least
 * c2v_corpus_text_scratch_bytes(rows) bytes for the rows of one call.  No engine handle is needed; failures return a
 * negative c2v_status with the message in c2v_last_error(NULL).  Asynchronous on `stream`. */
size_t c2v_corpus_text_scratch_bytes(int64_t rows);

/* n >= 1 rows of name scores, all arrays device memory: row r's name is names[name_off[r], name_off[r + 1]) (as
 * c2v_reader_eval_take writes them), its line `name\trank\tlogp\ttop1_name\ttop1_logp\n` from target / rank / logp / top1
 * / top1_logp [n] (c2v_name_scores' outputs for the targets).  A row whose target is `oov` prints '-' for its rank and
 * logp; rank 0 prints '-'.  top1_name is words[word_off[top1], word_off[top1 + 1]) (c2v_reader_eval_words), the OOV
 * word for a top1 outside [0, n_words). */
int c2v_name_scores_text(int32_t n, const char* names, const int64_t* name_off, const int32_t* target, int32_t oov,
                         const int32_t* rank, const float* logp, const int32_t* top1, const float* top1_logp,
                         const char* words, const int64_t* word_off, int32_t n_words, void* scratch, size_t scratch_bytes,
                         char* out, int64_t out_cap, int64_t* total, void* stream);

/* Lines [first, first + n) of a corpus of `rows` rows (rows < 2^31), all arrays device memory: row r's name is
 * names[name_off[r], name_off[r + 1]) (name_off [rows + 1]), its neighbours idx / val [rows, k] (c2v_knn_search's
 * outputs).  Line r is the name, then `\t<id>,<name of id>,<val>` for each neighbour in order; the INT_MAX padding
 * (any id outside [0, rows)) is skipped. */
int c2v_nearest_text(int64_t first, int64_t n, int64_t rows, int32_t k, const char* names, const int64_t* name_off,
                     const int32_t* idx, const float* val, void* scratch, size_t scratch_bytes, char* out, int64_t out_cap,
                     int64_t* total, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* C2V_B200_H_ */
