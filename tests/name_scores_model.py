"""Float64 statement of c2v_name_scores (DESIGN.md §6n, include/c2v_b200.h): each example's own name scored over its whole
logits row S_b [Y] (the special word at row 0 included), with target index y_b and t_b = S_b[y_b]:

  lse_b       = m_b + log sum_j exp(S_b[j] - m_b),  m_b = max_j S_b[j]
  rank_b      = 1 + #{j : S_b[j] > t_b} + #{j < y_b : S_b[j] == t_b}   (1-based, tf.nn.top_k's order)
  logp_b      = t_b - lse_b
  top1_b      = the lowest j with S_b[j] == m_b
  top1_logp_b = m_b - lse_b
A row holding a NaN: rank 0 and NaN log-probabilities; top1 is then the lowest index of the largest non-NaN logit, the
first id tf.nn.top_k's order gives when NaNs never enter it."""
from __future__ import annotations

import numpy as np


def name_scores64(S, y):
    """S [B, Y] logits (any float dtype, read as float64), y [B] target indices -> (rank [B] int64, logp [B],
    top1 [B] int64, top1_logp [B])."""
    S = np.asarray(S, dtype=np.float64)
    y = np.asarray(y, dtype=np.int64)
    B, Y = S.shape
    rank = np.zeros(B, dtype=np.int64)
    top1 = np.zeros(B, dtype=np.int64)
    logp = np.full(B, np.nan)
    top1_logp = np.full(B, np.nan)
    cols = np.arange(Y)
    for b in range(B):
        row = S[b]
        nan = np.isnan(row)
        finite = row[~nan]
        m = finite.max() if finite.size else -np.inf
        top1[b] = cols[~nan][np.argmax(finite == m)] if finite.size else np.iinfo(np.int32).max
        if nan.any():
            continue
        t = row[y[b]]
        rank[b] = 1 + int(np.sum(row > t)) + int(np.sum((row == t) & (cols < y[b])))
        lse = m + np.log(np.sum(np.exp(row - m)))
        logp[b] = t - lse
        top1_logp[b] = m - lse
    return rank, logp, top1, top1_logp
