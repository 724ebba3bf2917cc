"""A numpy statement of the sampled-softmax step on a row-sharded target table (DESIGN.md section 6j, "Several GPUs").

W ranks, rank r holding the contiguous block trainer.target_row_block(Y, r, W) of target rows and the examples
[r * Bl, (r + 1) * Bl) of the global batch.  Every rank has the same S negatives.  The step:
  pack   each owner writes the negatives' rows and the global batch's target rows that live in its block into zero-filled
         [S, D] / [Bt, D] buffers; the sum over ranks of the first (all-reduce) gives every rank all S rows, the sum of the
         second (reduce-scatter) the true rows of its own Bl examples.  Every element has exactly one owner.
  head   each rank, on its own examples: logits over {true, S negatives} minus logq, accidental hits masked, softmax,
         loss partial = sum_b loss_b / Bt, dl = (p - onehot) / Bt, dv = dl[:, 0] * true_row + dl[:, 1:] . neg_rows.
  partials  g_true [Bl, D] = dl[b, 0] v_b; g_neg [S, D] = sum over the rank's b of dl[b, 1+s] v_b in chunks of 64 examples.
  fold   the owner of a row stores, from 0 and in this order, g_true_all[b] for each global b whose target is the row, then
         g_neg_all[r][s] for each s holding the row and r = 0 .. W-1.  The loss is the partials added in rank order.
Every sum is written out in that order, so the statement runs in float32 or float64.
"""
from __future__ import annotations

import numpy as np

CHUNK = 64                       # examples per partial sum of g_neg (the deterministic sampled-softmax kernel's chunk)


def target_row_block(Y: int, rank: int, world: int):
    """code2vec_b200.trainer.target_row_block, restated: the contiguous rows [row0, row1) rank `rank` holds."""
    per = (Y + world - 1) // world
    row0 = min(rank * per, Y)
    return row0, min(row0 + per, Y)


def pack(Yt, ids, row0, row1):
    """[len(ids), D]: Yt[id] for the ids in [row0, row1), zeros elsewhere."""
    out = np.zeros((len(ids), Yt.shape[1]), dtype=Yt.dtype)
    own = (ids >= row0) & (ids < row1)
    out[own] = Yt[ids[own]]
    return out


def head(v, true_rows, neg_rows, target, sampled, logq_true, logq_sampled, Bt):
    """One rank's head on its examples: (loss partial, dl [Bl, 1+S], dv [Bl, D])."""
    dt = v.dtype.type
    l_true = (v * true_rows).sum(axis=1) - logq_true.astype(dt)
    l_samp = v @ neg_rows.T - logq_sampled.astype(dt)[None, :]
    hit = sampled[None, :] == target[:, None]
    l_samp = np.where(hit, dt(-1e9), l_samp)
    logits = np.concatenate([l_true[:, None], l_samp], axis=1)
    m = logits.max(axis=1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(logits - m).sum(axis=1))
    loss_partial = dt((lse - logits[:, 0]).sum() / dt(Bt))
    p = np.exp(logits - lse[:, None])
    p[:, 0] -= 1
    dl = p / dt(Bt)
    dl[:, 1:] = np.where(hit, dt(0), dl[:, 1:])
    dv = dl[:, :1] * true_rows + dl[:, 1:] @ neg_rows
    return loss_partial, dl, dv


def partials(v, dl):
    """(g_true [Bl, D], g_neg [S, D]) of one rank."""
    g_true = dl[:, :1] * v
    g_neg = np.zeros((dl.shape[1] - 1, v.shape[1]), dtype=v.dtype)
    for b0 in range(0, v.shape[0], CHUNK):
        g_neg = g_neg + dl[b0:b0 + CHUNK, 1:].T @ v[b0:b0 + CHUNK]
    return g_true, g_neg


def fold(g_true_all, g_neg_all, target_all, sampled, row0, row1):
    """The owner's gradient block [row1 - row0, D]: rows nobody references stay zero."""
    D = g_true_all.shape[1]
    out = np.zeros((row1 - row0, D), dtype=g_true_all.dtype)
    for row in dict.fromkeys(np.concatenate([target_all, sampled]).tolist()):       # first occurrences, in list order
        if not row0 <= row < row1:
            continue
        acc = np.zeros(D, dtype=g_true_all.dtype)
        for b in np.flatnonzero(target_all == row):
            acc = acc + g_true_all[b]
        for s in np.flatnonzero(sampled == row):
            for r in range(g_neg_all.shape[0]):
                acc = acc + g_neg_all[r, s]
        out[row - row0] = acc
    return out


def step(Yt, v, target, sampled, logq_true, logq_sampled, world):
    """The W-rank step on the global batch v [Bt, D] / target [Bt] (Bt a multiple of world): (loss, dv [Bt, D], the
    assembled target gradient [Y, D], the per-rank loss partials)."""
    Y, D = Yt.shape
    Bt = len(target)
    assert Bt % world == 0
    Bl = Bt // world
    blocks = [target_row_block(Y, r, world) for r in range(world)]
    owners = np.zeros(Y, dtype=np.int64)
    for r0, r1 in blocks:
        owners[r0:r1] += 1
    assert (owners == 1).all(), "every target row has exactly one owner"
    neg_send = [pack(Yt, sampled, r0, r1) for r0, r1 in blocks]
    true_send = [pack(Yt, target, r0, r1) for r0, r1 in blocks]
    # one contributor per row: the sums are exact in any order
    for ids in (sampled, target):
        assert (sum((ids >= r0) & (ids < r1) for r0, r1 in blocks) == 1).all()
    neg = np.sum(neg_send, axis=0)
    true_all = np.sum(true_send, axis=0)
    parts, dv, g_true, g_neg = [], [], [], []
    for r in range(world):
        ex = slice(r * Bl, (r + 1) * Bl)
        lp, dl, dv_r = head(v[ex], true_all[ex], neg, target[ex], sampled, logq_true[ex], logq_sampled, Bt)
        gt, gn = partials(v[ex], dl)
        parts.append(lp)
        dv.append(dv_r)
        g_true.append(gt)
        g_neg.append(gn)
    g_true_all, g_neg_all = np.concatenate(g_true), np.stack(g_neg)
    g_tgt = np.zeros_like(Yt)
    for r0, r1 in blocks:
        g_tgt[r0:r1] = fold(g_true_all, g_neg_all, target, sampled, r0, r1)
    loss = v.dtype.type(0)
    for lp in parts:
        loss = loss + lp
    return loss, np.concatenate(dv), g_tgt, np.array(parts)
