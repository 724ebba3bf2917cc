"""Train-step driver over one PathAttentionEngine per process (one process per GPU).

Single GPU: one C-ABI call per batch (c2v_train_batch_host == the reference's
``sess.run([optimizer, train_loss])``, tensorflow_model.py:80).

Data parallel (BASELINE config 4; the reference has no multi-GPU path, SURVEY section 2.2): the
batch is sharded across ranks and the tables are replicated.  Two interchangeable schedules, both
leaving every replica with bit-identical parameters:

  "allreduce" : all-reduce(mean) of the five gradient tensors, then the full Adam on every rank.
  "sharded"   : (default) the model lives in one flat buffer split into two buckets -- A = the
                target table, whose gradient is complete right after the dY GEMM, B = the rest.
                Each bucket is reduce-scattered (mean) so that rank r owns 1/world of it, Adam runs
                on the owned slices only (c2v_adam_step_range: 1/world of the 9.2 GB optimizer
                traffic), and the updated slices are all-gathered back.  Bucket A's
                reduce-scatter is issued on a side stream as soon as the engine's
                "target_grads_ready" event fires, so it overlaps the context backward pass.

  "table_sharded" : (default on 2/4/8 GPUs) as "sharded" for the target table, but the two embedding
                tables are not replicated at all: they are row-sharded over the ranks and reached
                through peer memory (PathAttentionEngine.enable_table_sharding).  The forward gather
                loads rows from the owning GPU over NVLink and the backward scatter-add issues
                red.global.add to it, so no embedding gradient is ever reduced or gathered (1.13 GB
                of the 1.53 GB per step disappears from the collectives) and each rank's Adam
                touches 1/world of every table.  Ordering comes from the collectives that remain:
                the all-reduce of the TRANSFORM/ATTENTION gradients is issued after the local
                scatter, so its completion means every rank's scatter has landed (Adam may run);
                the all-gather of the updated target table is issued after the local Adam, so its
                completion means every shard is updated (the next gather may run).

  "fully_sharded" : (BASELINE config 5) nothing big is replicated.  Embedding tables as in
                "table_sharded"; the target table is row-sharded in contiguous blocks and each rank's
                engine is built for its LOCAL target rows and the GLOBAL batch (make_fully_sharded_engine).
                A step is phase-split (c2v_context_forward / c2v_target_forward / c2v_lse_combine /
                c2v_target_backward / c2v_context_backward) and moves only small tensors between the
                phases: all-gather of code vectors [Bt, D] and targets, all-gather of the per-row
                (max, sum exp) partials and all-reduce of the true logits [Bt], reduce-scatter of dv
                [Bt, D].  No logits slab and no table gradient ever crosses NVLink; each rank's Adam
                covers 1/world of all three tables.
                In the tensor-core modes the per-row partials are (c, sum exp(s - c)) of the exp_slab
                schedule (c = the true logit on the rank that owns the class, 0 elsewhere) -- the same
                combine formula -- and the softmax's normalisation is applied as per-row factors inside
                the two gradient GEMMs (DESIGN.md section 4.9).  Trainer(allow_single_rank=True) keeps
                this schedule in a process group of ONE rank, so a one-GPU box can run the whole path
                (tests/test_gpu_dp.py).

torch.distributed (NCCL over NVLink/NVSwitch; gloo in the CPU tests of the host logic) is plumbing;
all arithmetic stays in the engine's kernels.
"""
from __future__ import annotations

from typing import Optional

import numpy as np

from .engine import PARAM_NAMES, PathAttentionEngine

ADAM_DEFAULTS = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8)   # tf.compat.v1.train.AdamOptimizer()


def _dist():
    import torch.distributed as dist
    return dist


def allreduce_mean_(tensors, group=None):
    """In-place mean over ranks of each tensor in `tensors` (list).  NCCL averages in the
    collective itself; gloo (CPU tests) sums and scales."""
    dist = _dist()
    if not (dist.is_available() and dist.is_initialized()):
        return
    world = dist.get_world_size(group)
    if world == 1:
        return
    backend = dist.get_backend(group)
    op = dist.ReduceOp.AVG if backend == "nccl" else dist.ReduceOp.SUM
    handles = [dist.all_reduce(t, op=op, group=group, async_op=True) for t in tensors]
    for h in handles:
        h.wait()
    if backend != "nccl":
        for t in tensors:
            t.mul_(1.0 / world)


def reduce_scatter_mean(out_shard, flat, group=None, async_op=False):
    """out_shard <- mean over ranks of this rank's 1/world slice of `flat` (len(flat) % world == 0)."""
    dist = _dist()
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    if dist.get_backend(group) == "nccl":
        return dist.reduce_scatter_tensor(out_shard, flat, op=dist.ReduceOp.AVG, group=group, async_op=async_op)
    # gloo has no reduce-scatter: all-reduce a copy and keep the owned slice (CPU tests only)
    tmp = flat.clone()
    dist.all_reduce(tmp, op=dist.ReduceOp.SUM, group=group)
    n = flat.numel() // world
    out_shard.copy_(tmp[rank * n:(rank + 1) * n] / world)
    return None


def all_gather_flat(flat, shard, group=None, async_op=False):
    """flat <- concatenation over ranks of `shard` (len(flat) == world * len(shard))."""
    dist = _dist()
    if dist.get_backend(group) == "nccl":
        return dist.all_gather_into_tensor(flat, shard, group=group, async_op=async_op)
    world = dist.get_world_size(group)
    n = shard.numel()
    parts = [flat[i * n:(i + 1) * n] for i in range(world)]
    dist.all_gather(parts, shard.clone(), group=group)
    return None


def target_row_block(n_targets: int, rank: int, world: int):
    """Contiguous block [row0, row1) of target-table rows owned by `rank` in the fully sharded schedule."""
    per = (n_targets + world - 1) // world
    row0 = min(rank * per, n_targets)
    return row0, min(row0 + per, n_targets)


def make_fully_sharded_engine(dims, local_batch: int, device: int, group=None, training: bool = True):
    """Engine for the fully sharded schedule: `dims` are the GLOBAL model dims (EngineDims); the returned
    engine holds this rank's block of target rows and is sized for the global batch."""
    from dataclasses import replace
    dist = _dist()
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    # the last rank's block is the smallest: when it is empty, some rank has no target rows, and an engine needs at
    # least one, whose logit would then enter every example's normaliser.  Every rank refuses alike.
    last0, last1 = target_row_block(dims.target_vocab, world - 1, world)
    if last1 <= last0:
        per = (dims.target_vocab + world - 1) // world
        raise ValueError("fully_sharded: %d target rows in blocks of %d leave ranks %d..%d of %d without a row"
                         % (dims.target_vocab, per, -(-dims.target_vocab // per), world - 1, world))
    row0, row1 = target_row_block(dims.target_vocab, rank, world)
    local = replace(dims, target_vocab=row1 - row0, max_batch=local_batch * world)
    eng = PathAttentionEngine(local, device=device, training=training)
    eng.global_target_vocab, eng.target_row0, eng.local_batch = dims.target_vocab, row0, local_batch
    return eng


def deterministic_refusal(schedule: str, world: int, push_grads: bool, ordered_exchange: bool = False) -> Optional[str]:
    """Why `schedule` on `world` ranks cannot run with the engine option "deterministic", or None if it can.  The option
    fixes the order of every reduction into tables the engine holds itself; row-sharded tables over several ranks take
    order-free cross-rank red.adds (or inbox folds) unless ordered_exchange sends sorted per-row sums that the owners
    fold in rank order.  NCCL's own reduction order (allreduce / sharded) is outside it."""
    if schedule in ("table_sharded", "fully_sharded") and world > 1 and not ordered_exchange:
        if push_grads:
            return ("deterministic training is not available with the %s schedule on %d ranks: peers push embedding "
                    "gradients into a scatter inbox that is folded with atomics" % (schedule, world))
        return ("deterministic training is not available with the %s schedule on %d ranks: the embedding tables are "
                "row-sharded and peers red.add into them in no fixed order" % (schedule, world))
    return None


def shard_bounds(n: int, rank: int, world: int):
    """Contiguous slice [lo, hi) of n items owned by `rank` (sizes differ by at most 1)."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class Trainer:
    def __init__(self, engine: PathAttentionEngine, keep_prob: float = 0.75, seed: int = 0, group=None,
                 adam: Optional[dict] = None, schedule: str = "table_sharded", lazy_adam: bool = True,
                 fuse_target_adam: bool = True, push_grads: bool = False, allow_single_rank: bool = False,
                 deterministic: bool = False, ordered_exchange: bool = False):
        self.e = engine
        self.keep = float(keep_prob)
        self.seed = int(seed)
        self.group = group
        self.adam = dict(ADAM_DEFAULTS, **(adam or {}))
        torch = engine.torch
        dist = _dist()
        grouped = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if grouped else 1
        self.rank = dist.get_rank(group) if self.world > 1 else 0
        # allow_single_rank: keep the fully sharded schedule (IPC-homed tables, phase-split entry points, collectives) in a
        # process group of ONE rank -- no use in production, but it lets a one-GPU box run that whole code path
        self.multi = self.world > 1 or (allow_single_rank and grouped and schedule == "fully_sharded")
        self.schedule = schedule if self.multi else "single"
        if self.schedule in ("table_sharded", "fully_sharded") and self.world not in (1, 2, 4, 8):
            self.schedule = "sharded"
        # deterministic: every step's results depend only on its inputs, seeds and options (engine option "deterministic")
        # ordered_exchange: the row-sharded schedules send embedding gradients as sorted per-row sums through the scatter
        # inbox and the owners fold them in rank order (engine option "ordered_exchange"); deterministic needs it there
        self.deterministic = bool(deterministic)
        if self.deterministic:
            why = deterministic_refusal(self.schedule, self.world, push_grads, ordered_exchange)
            if why:
                raise ValueError(why + "; pass ordered_exchange=True")
        if self.schedule == "fully_sharded":
            if not hasattr(engine, "target_row0"):
                raise ValueError("the fully_sharded schedule needs an engine from make_fully_sharded_engine()")
            with torch.cuda.device(engine.dev):
                engine.enable_table_sharding(group, push_grads=push_grads, ordered_exchange=ordered_exchange)
            engine.set_option("grad_scale_inverse", 1)     # dv already carries the 1/global-batch factor
            Bl, Bt, D = engine.local_batch, engine.local_batch * self.world, engine.dims.code_dim
            f32, i32, dev = torch.float32, torch.int32, engine.dev
            z = lambda shape, dt=f32: torch.zeros(shape, dtype=dt, device=dev)
            self._fs = dict(v_local=z((Bl, D)), v_all=z((Bt, D)), tgt_all=z((Bt,), i32), rmax=z((Bt,)), rsum=z((Bt,)),
                            tlogit=z((Bt,)), maxes=z((self.world, Bt)), sums=z((self.world, Bt)), lse=z((Bt,)),
                            dv_part=z((Bt, D)), dv_local=z((Bl, D)), loss=z((1,)), token=z((1,)))
            # predict(): this rank's candidates, every rank's (all-gathered), and the merged rows of its own examples
            W, k = self.world, min(engine.dims.top_k, engine.global_target_vocab)
            self._pred = dict(idx=z((Bt, k), i32), val=z((Bt, k)), idx_all=z((W, Bt, k), i32), val_all=z((W, Bt, k)),
                              idx_out=z((Bl, k), i32), val_out=z((Bl, k)))
            layout, total = engine.flat_layout()
            small0 = [off for k, off, n in layout if k == "W"][0]
            self._small = (small0, total)
        B, C = engine.dims.max_batch, engine.dims.max_contexts
        self._dev = None
        if self.multi:
            i32, f32 = torch.int32, torch.float32
            self._dev = dict(src=torch.empty((B, C), dtype=i32, device=engine.dev),
                             path=torch.empty((B, C), dtype=i32, device=engine.dev),
                             tgt=torch.empty((B, C), dtype=i32, device=engine.dev),
                             mask=torch.empty((B, C), dtype=f32, device=engine.dev),
                             target=torch.empty((B,), dtype=i32, device=engine.dev))
        if self.schedule == "table_sharded":
            with torch.cuda.device(engine.dev):
                engine.enable_table_sharding(group, push_grads=push_grads, ordered_exchange=ordered_exchange)
            (a0, a1), _ = engine.bucket_bounds()
            layout, total = engine.flat_layout()
            small0 = [off for k, off, n in layout if k == "W"][0]         # W, a: the tail of the flat buffer
            w, r = self.world, self.rank
            na = (a1 - a0) // w
            self._bucket = [(a0, a1, a0 + r * na, a0 + (r + 1) * na)]
            self._small = (small0, total)
            self._gshard = [torch.empty(na, dtype=torch.float32, device=engine.dev)]
            self._side = torch.cuda.Stream(device=engine.dev)
            self._ev_tgt = torch.cuda.Event()
            with torch.cuda.device(engine.dev):
                engine.set_event("target_grads_ready", self._ev_tgt)
        if self.schedule in ("sharded", "table_sharded"):
            engine.set_option("dy_late", 0)     # these schedules start the target table's reduce-scatter right after dY
        if self.schedule == "sharded":
            (a0, a1), (b0, b1) = engine.bucket_bounds()
            w, r = self.world, self.rank
            assert (a1 - a0) % w == 0 and (b1 - b0) % w == 0
            na, nb = (a1 - a0) // w, (b1 - b0) // w
            self._bucket = [(a0, a1, a0 + r * na, a0 + (r + 1) * na), (b0, b1, b0 + r * nb, b0 + (r + 1) * nb)]
            self._gshard = [torch.empty(na, dtype=torch.float32, device=engine.dev),
                            torch.empty(nb, dtype=torch.float32, device=engine.dev)]
            self._side = torch.cuda.Stream(device=engine.dev)
            self._ev_tgt = torch.cuda.Event()
            with torch.cuda.device(engine.dev):
                engine.set_event("target_grads_ready", self._ev_tgt)
        if self.schedule == "single" and lazy_adam and engine.training:
            engine.set_option("lazy_adam", 1)       # exact, see c2v_b200.h; the multi-GPU schedules stay dense
        # target-table Adam inside the dY epilogue (bit-identical, see c2v_arm_target_adam): wherever the
        # target gradient is complete on this rank without a collective
        self.fuse_tgt = bool(fuse_target_adam) and self.schedule in ("single", "fully_sharded") and engine.training
        if self.schedule == "single":
            engine.set_option("fuse_target_adam", 1 if self.fuse_tgt else 0)     # for train_batch_host
            # dY (+ the target table's Adam step) straight after dv: on one GPU it is HBM-bound like the scatter-add
            # it would otherwise share the memory system with (dy_late 0/1/2 all measure within 1 %)
            engine.set_option("dy_late", 0)
        engine.set_option("deterministic", 1 if self.deterministic else 0)
        self._loss_host = torch.zeros(1, dtype=torch.float32).pin_memory()

    # ---- inputs already resident on the device ----------------------------------------------
    def step_device(self, src, path, tgt, mask, target, next_batch=None):
        """Forward+backward, gradient exchange, Adam.  Returns the device loss tensor (no sync).
        next_batch: optional (src, path, tgt) device tensors of the batch the NEXT call will get -- with lazy
        Adam the deferred updates of its rows then overlap this step's backward GEMMs (c2v_hint_next_batch)."""
        if self.schedule == "fully_sharded":
            return self._fully_sharded_step(src, path, tgt, mask, target)
        e = self.e
        t = e.adam_t + 1
        if self.fuse_tgt:
            e.arm_target_adam(t, **self.adam)
            if next_batch is not None and self.schedule == "single":
                e.hint_next_batch(*next_batch[:3])
        # dropout stream position (seed, t); replicas use different seeds so their masks differ
        loss = e.train_step(src, path, tgt, mask, target, keep=self.keep, seed=self.seed + self.rank, step=t)
        if self.schedule == "single":
            e.adam_step(t=t, **self.adam)
        elif self.schedule == "allreduce":
            allreduce_mean_([e.grads[k] for k in PARAM_NAMES], self.group)
            e.adam_step(t=t, **self.adam)
        elif self.schedule == "table_sharded":
            self._table_sharded_update(t)
        elif self.schedule == "fully_sharded":
            raise RuntimeError("fully_sharded uses step_device_fully_sharded (phase-split step)")
        else:
            self._sharded_update(t)
        return loss

    def step_ring(self, ring, rows: int, loss_out):
        """One training step on the next filled slot of a PinnedBatchRing, fully asynchronous (single GPU)."""
        if self.schedule != "single":
            raise RuntimeError("step_ring is single-GPU")
        ring.submit_next(self.e, rows, loss_out, keep=self.keep, seed=self.seed, **self.adam)

    def step_device_sampled(self, src, path, tgt, mask, target, sampled, logq_true, logq_sampled):
        """BASELINE config 3: one training step with the sampled softmax (c2v_sampled_train_step) + Adam.  Single
        GPU.  With lazy Adam the target table's rows are updated lazily too (only the B + S rows the step reads)."""
        if self.schedule != "single":
            raise RuntimeError("the sampled-softmax step is single-GPU")
        e = self.e
        t = e.adam_t + 1
        loss = e.sampled_train_step(src, path, tgt, mask, target, sampled, logq_true, logq_sampled, keep=self.keep,
                                    seed=self.seed, step=t)
        e.adam_step(t=t, **self.adam)
        return loss

    def step_sampled(self, src, path, tgt, mask, target, num_sampled: int):
        """One sampled-softmax training step whose num_sampled negatives are drawn on the device for (seed, t = adam_t + 1)
        (c2v_sample_log_uniform, DESIGN.md section 6j), then step_device_sampled.  Returns the device loss without a sync.
        The draw depends on the step count only, so a run resumed from a checkpoint (which restores adam_t) continues the
        same negatives.  One GPU, or the fully sharded schedule (_fully_sharded_sampled_step): there every rank draws
        the negatives of the one-GPU run with the same seed over the global vocabulary."""
        if self.schedule == "fully_sharded":
            return self._fully_sharded_sampled_step(src, path, tgt, mask, target, int(num_sampled))
        if self.schedule != "single":
            raise RuntimeError("the sampled-softmax step runs on one GPU or on the fully_sharded schedule, not on %r"
                               % self.schedule)
        e = self.e
        sampled, lq_t, lq_s, _ = e.sample_log_uniform(target, num_sampled, self.seed, e.adam_t + 1)
        return self.step_device_sampled(src, path, tgt, mask, target, sampled, lq_t, lq_s)

    def step_host_sampled(self, src, path, tgt, mask, target, num_sampled: int) -> float:
        """step_sampled on HOST buffers (numpy / pinned tensors): uploads them, steps and returns the loss (synchronises)."""
        e = self.e
        torch = e.torch
        if self._dev is None:
            Bm, Cm = e.dims.max_batch, e.dims.max_contexts
            z = lambda shape, dt: torch.empty(shape, dtype=dt, device=e.dev)
            self._dev = dict(src=z((Bm, Cm), torch.int32), path=z((Bm, Cm), torch.int32), tgt=z((Bm, Cm), torch.int32),
                             mask=z((Bm, Cm), torch.float32), target=z((Bm,), torch.int32))
        B = int(src.shape[0])
        d = self._dev
        for name, arr in (("src", src), ("path", path), ("tgt", tgt), ("mask", mask), ("target", target)):
            t = arr if isinstance(arr, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(arr))
            d[name][:B].copy_(t, non_blocking=True)
        loss = self.step_sampled(d["src"][:B], d["path"][:B], d["tgt"][:B], d["mask"][:B], d["target"][:B], num_sampled)
        self._loss_host.copy_(loss, non_blocking=True)
        torch.cuda.current_stream(e.dev).synchronize()
        return float(self._loss_host[0])

    def predict(self, src, path, tgt, mask, normalize: int = 0):
        """Top-k prediction of this rank's examples: (idx [B, k], val [B, k], code_vec [B, D]) as device tensors, the
        result of forward + topk on one engine holding the whole model (normalize as c2v_topk).  No training state is
        touched, so it runs between training steps and on engines made with training=False.
        fully_sharded: the rank's engine holds one block of target rows, so the code vectors are all-gathered, every
        rank ranks its block for the whole global batch (c2v_topk_partial), the [Bt, k] candidates (and for normalize 2
        the per-row (max, sum exp)) are all-gathered, and each rank merges the rows of its own examples
        (c2v_topk_merge).  The returned tensors are buffers the next predict() call overwrites."""
        e = self.e
        if self.schedule != "fully_sharded":
            code, _ = e.forward(src, path, tgt, mask, want_attention=False)
            idx, val = e.topk(code, normalize)
            return idx, val, code
        dist = _dist()
        Bl = int(src.shape[0])
        fs, pr = self._fs_views(Bl), self._pred_views(Bl)
        full = normalize == 2
        e.forward(src, path, tgt, mask, want_attention=False, code_out=fs["v_local"])
        dist.all_gather_into_tensor(fs["v_all"], fs["v_local"], group=self.group)
        k = pr["idx"].shape[1]
        e.topk_partial(fs["v_all"], e.target_row0, k, pr["idx"], pr["val"], fs["rmax"] if full else None,
                       fs["rsum"] if full else None)
        dist.all_gather_into_tensor(pr["idx_all"].view(-1), pr["idx"].view(-1), group=self.group)
        dist.all_gather_into_tensor(pr["val_all"].view(-1), pr["val"].view(-1), group=self.group)
        if full:
            dist.all_gather_into_tensor(fs["maxes"].view(-1), fs["rmax"], group=self.group)
            dist.all_gather_into_tensor(fs["sums"].view(-1), fs["rsum"], group=self.group)
        e.topk_merge(pr["idx_all"], pr["val_all"], fs["maxes"] if full else None, fs["sums"] if full else None,
                     self.rank * Bl, Bl, normalize, pr["idx_out"], pr["val_out"])
        return pr["idx_out"], pr["val_out"], fs["v_local"]

    def _local_batch(self, B: int):
        if not 0 < B <= self.e.local_batch:
            raise ValueError("fully_sharded takes 1 to %d rows per rank (the engine's local batch), the same number on "
                             "every rank; got %d" % (self.e.local_batch, B))

    def _fs_views(self, B: int):
        """The step's buffers for a local batch of B <= local_batch rows (the same B on every rank): the [Bl] / [Bt]
        buffers as leading views, the [W, Bt] ones as contiguous [W, B * W] views of their first elements."""
        self._local_batch(B)
        fs = self._fs
        if B == self.e.local_batch:
            return fs
        W, Bt = self.world, B * self.world
        v = dict(fs)
        for name in ("v_local", "dv_local"):
            v[name] = fs[name][:B]
        for name in ("v_all", "tgt_all", "rmax", "rsum", "tlogit", "lse", "dv_part"):
            v[name] = fs[name][:Bt]
        for name in ("maxes", "sums"):
            v[name] = fs[name].view(-1)[:W * Bt].view(W, Bt)
        return v

    def _pred_views(self, B: int):
        """predict()'s buffers for a local batch of B rows, as _fs_views."""
        pr = self._pred
        if B == self.e.local_batch:
            return pr
        W, Bt, k = self.world, B * self.world, pr["idx"].shape[1]
        v = dict(idx=pr["idx"][:Bt], val=pr["val"][:Bt], idx_out=pr["idx_out"][:B], val_out=pr["val_out"][:B])
        for name in ("idx_all", "val_all"):
            v[name] = pr[name].view(-1)[:W * Bt * k].view(W, Bt, k)
        return v

    def _fully_sharded_step(self, src, path, tgt, mask, target):
        e, dist = self.e, _dist()
        t = e.adam_t + 1
        fs = self._fs_views(int(src.shape[0]))
        seed = self.seed + self.rank
        e.context_forward(src, path, tgt, mask, fs["v_local"], keep=self.keep, seed=seed, step=t)
        dist.all_gather_into_tensor(fs["v_all"], fs["v_local"], group=self.group)
        dist.all_gather_into_tensor(fs["tgt_all"], target, group=self.group)
        e.target_forward(fs["v_all"], fs["tgt_all"], e.target_row0, fs["rmax"], fs["rsum"], fs["tlogit"])
        dist.all_gather_into_tensor(fs["maxes"].view(-1), fs["rmax"], group=self.group)
        dist.all_gather_into_tensor(fs["sums"].view(-1), fs["rsum"], group=self.group)
        dist.all_reduce(fs["tlogit"], op=dist.ReduceOp.SUM, group=self.group)
        e.lse_combine(fs["maxes"], fs["sums"], fs["tlogit"], fs["lse"], fs["loss"])
        if self.fuse_tgt:
            e.arm_target_adam(t, **self.adam)
        e.target_backward(fs["v_all"], fs["lse"], fs["tgt_all"], e.target_row0, fs["dv_part"])
        dist.reduce_scatter_tensor(fs["dv_local"], fs["dv_part"], op=dist.ReduceOp.SUM, group=self.group)
        e.context_backward(src, path, tgt, mask, fs["dv_local"], keep=self.keep, seed=seed, step=t)
        self._fully_sharded_update(t)
        return fs["loss"]

    def _sampled_views(self, B: int, S: int):
        """The sampled step's buffers for a local batch of B rows and S negatives (allocated for the engine's local batch
        at the first call with this S): packed rows, partial target gradients and loss partials."""
        e, torch = self.e, self.e.torch
        buf = getattr(self, "_fss", None)
        if buf is None or buf["S"] != S:
            W, Bl, D = self.world, e.local_batch, e.dims.code_dim
            z = lambda *shape: torch.zeros(shape, dtype=torch.float32, device=e.dev)
            buf = self._fss = dict(S=S, neg=z(S, D), true_send=z(W * Bl, D), true=z(Bl, D), g_neg=z(S, D),
                                   g_neg_all=z(W, S, D), g_true=z(Bl, D), g_true_all=z(W * Bl, D), loss_part=z(1),
                                   loss_parts=z(W))
        if B == e.local_batch:
            return buf
        v = dict(buf)
        for name in ("true", "g_true"):
            v[name] = buf[name][:B]
        for name in ("true_send", "g_true_all"):
            v[name] = buf[name][:B * self.world]
        return v

    def _fully_sharded_sampled_step(self, src, path, tgt, mask, target, S: int):
        """The sampled-softmax step of the fully sharded schedule (DESIGN.md section 6j): the rows move to the examples.
        Every rank draws the same S negatives over the global vocabulary for (self.seed, t); the owners pack those rows
        and their block's rows of the Bt targets (one all-reduce and one reduce-scatter, each element with one non-zero
        contributor, so both exact); each rank runs the head on its own examples, and the partial target gradients are
        all-gathered and folded by the owners in a fixed order.  The dY-epilogue Adam is not armed: the target block
        takes the dense Adam of _fully_sharded_update."""
        e, dist = self.e, _dist()
        if not getattr(self, "_seed_agreed", False):
            # the packed rows are summed over ranks: a rank that drew other negatives would add rows of other ids
            seeds = [None] * self.world
            dist.all_gather_object(seeds, self.seed, group=self.group)
            if len(set(seeds)) > 1:
                raise ValueError("the sampled-softmax step on the fully_sharded schedule needs the same Trainer seed on "
                                 "every rank (every rank draws the same negatives from it); got seeds %s" % seeds)
            self._seed_agreed = True
        t = e.adam_t + 1
        Bl = int(src.shape[0])
        fs, ss = self._fs_views(Bl), self._sampled_views(Bl, S)
        seed = self.seed + self.rank
        e.context_forward(src, path, tgt, mask, fs["v_local"], keep=self.keep, seed=seed, step=t)
        dist.all_gather_into_tensor(fs["tgt_all"], target, group=self.group)
        sampled, lq_t, lq_s, _ = e.sample_log_uniform_vocab(target, S, e.global_target_vocab, self.seed, t)
        e.sampled_pack_rows(sampled, fs["tgt_all"], e.target_row0, ss["neg"], ss["true_send"])
        dist.all_reduce(ss["neg"], op=dist.ReduceOp.SUM, group=self.group)
        dist.reduce_scatter_tensor(ss["true"], ss["true_send"], op=dist.ReduceOp.SUM, group=self.group)
        e.sampled_target_step(fs["v_local"], target, sampled, lq_t, lq_s, ss["neg"], ss["true"], 1.0 / (Bl * self.world),
                              fs["dv_local"], ss["g_true"], ss["g_neg"], ss["loss_part"])
        dist.all_gather_into_tensor(ss["g_neg_all"], ss["g_neg"], group=self.group)
        dist.all_gather_into_tensor(ss["g_true_all"], ss["g_true"], group=self.group)
        dist.all_gather_into_tensor(ss["loss_parts"], ss["loss_part"], group=self.group)
        e.sampled_target_fold(ss["g_true_all"], ss["g_neg_all"], fs["tgt_all"], sampled, e.target_row0, ss["loss_parts"],
                              fs["loss"])
        e.context_backward(src, path, tgt, mask, fs["dv_local"], keep=self.keep, seed=seed, step=t)
        self._fully_sharded_update(t)
        return fs["loss"]

    def _fully_sharded_update(self, t: int):
        """The fully sharded step's tail: the small gradients, the inbox fold and Adam on this rank's shards."""
        e, dist = self.e, _dist()
        fs = self._fs
        s0, s1 = self._small
        # sum (not mean): dv already carries 1/global batch.  Completion == every rank's scatter-add has landed.
        dist.all_reduce(e.flat_grads[s0:s1], op=dist.ReduceOp.SUM, group=self.group)
        if getattr(e, "push_grads", False):
            e.apply_scatter_inbox()          # every peer's rows have landed in this rank's inbox: fold them into the shards
        for name in ("tok", "path"):
            e.adam_step_range(e.shard_params[name], e.shard_grads[name], e.shard_m[name], e.shard_v[name], t,
                              zero_grad=True, **self.adam)
        if e.get_option("target_adam_fused_step") == t:
            e.set_option("target_adam_fused_step", 0)       # the dY epilogue already applied this rank's target rows
        else:
            e.adam_step_range(e.params["tgt"], e.grads["tgt"], e.adam_m["tgt"], e.adam_v["tgt"], t, **self.adam)
        e.adam_step_range(e.flat_params[s0:s1], e.flat_grads[s0:s1], e.flat_m[s0:s1], e.flat_v[s0:s1], t, **self.adam)
        # every shard must be updated before any rank's next gather reads it
        dist.all_reduce(fs["token"], group=self.group)

    def _table_sharded_update(self, t: int):
        e, torch = self.e, self.e.torch
        dist = _dist()
        main = torch.cuda.current_stream(e.dev)
        (a0, a1, alo, ahi), = self._bucket
        s0, s1 = self._small
        self._side.wait_event(self._ev_tgt)
        with torch.cuda.stream(self._side):
            wa = reduce_scatter_mean(self._gshard[0], e.flat_grads[a0:a1], self.group, async_op=True)
        # TRANSFORM / ATTENTION gradients (0.6 MB): mean over ranks; issued after the local scatter-add, so
        # its completion also tells this rank that every peer's red.adds into its shards have landed
        ws = dist.all_reduce(e.flat_grads[s0:s1], op=dist.ReduceOp.AVG, group=self.group, async_op=True)
        ws.wait()
        if getattr(e, "push_grads", False):
            e.apply_scatter_inbox()
        for name in ("tok", "path"):
            e.adam_step_range(e.shard_params[name], e.shard_grads[name], e.shard_m[name], e.shard_v[name], t,
                              zero_grad=True, **self.adam)
        e.adam_step_range(e.flat_params[s0:s1], e.flat_grads[s0:s1], e.flat_m[s0:s1], e.flat_v[s0:s1], t, **self.adam)
        if wa is not None:
            wa.wait()
        main.wait_stream(self._side)
        e.adam_step_range(e.flat_params[alo:ahi], self._gshard[0], e.flat_m[alo:ahi], e.flat_v[alo:ahi], t, **self.adam)
        # issued after every local Adam launch: completion == all ranks' shards are updated
        ga = all_gather_flat(e.flat_params[a0:a1], e.flat_params[alo:ahi], self.group, async_op=True)
        if ga is not None:
            ga.wait()

    def _sharded_update(self, t: int):
        e, torch = self.e, self.e.torch
        main = torch.cuda.current_stream(e.dev)
        (a0, a1, alo, ahi), (b0, b1, blo, bhi) = self._bucket
        # bucket A: may start as soon as dY is done (event recorded inside c2v_train_step)
        self._side.wait_event(self._ev_tgt)
        with torch.cuda.stream(self._side):
            wa = reduce_scatter_mean(self._gshard[0], e.flat_grads[a0:a1], self.group, async_op=True)
        wb = reduce_scatter_mean(self._gshard[1], e.flat_grads[b0:b1], self.group, async_op=True)
        for wk in (wa, wb):
            if wk is not None:
                wk.wait()                       # current (main) stream waits for the collective
        main.wait_stream(self._side)
        e.adam_step_range(e.flat_params[alo:ahi], self._gshard[0], e.flat_m[alo:ahi], e.flat_v[alo:ahi], t, **self.adam)
        e.adam_step_range(e.flat_params[blo:bhi], self._gshard[1], e.flat_m[blo:bhi], e.flat_v[blo:bhi], t, **self.adam)
        ga = all_gather_flat(e.flat_params[a0:a1], e.flat_params[alo:ahi], self.group, async_op=True)
        gb = all_gather_flat(e.flat_params[b0:b1], e.flat_params[blo:bhi], self.group, async_op=True)
        for wk in (ga, gb):
            if wk is not None:
                wk.wait()

    # ---- inputs in host memory (what train() does per batch) ---------------------------------
    def step_host(self, src, path, tgt, mask, target, next_batch=None) -> float:
        """One training step on HOST buffers (numpy / pinned tensors); returns the loss (synchronises).
        next_batch: optional host (src, path, tgt) of the following batch (see step_device)."""
        e = self.e
        if not self.multi:
            if next_batch is not None and self.fuse_tgt:
                e.hint_next_batch_host(*next_batch[:3])
            return e.train_batch_host(src, path, tgt, mask, target, keep=self.keep, seed=self.seed, **self.adam)
        torch = e.torch
        B = int(src.shape[0])
        d = self._dev
        for name, arr in (("src", src), ("path", path), ("tgt", tgt), ("mask", mask), ("target", target)):
            t = arr if isinstance(arr, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(arr))
            d[name][:B].copy_(t, non_blocking=True)
        loss = self.step_device(d["src"][:B], d["path"][:B], d["tgt"][:B], d["mask"][:B], d["target"][:B])
        self._loss_host.copy_(loss, non_blocking=True)
        torch.cuda.current_stream(e.dev).synchronize()
        return float(self._loss_host[0])
