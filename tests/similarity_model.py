"""Float64 statement of the nearest-neighbour search (DESIGN.md §6h, code2vec_b200/similarity.py), and a numpy model of
how the device computes it, for the tests.

  query64 / scores64 / search64 : gensim 4's KeyedVectors.most_similar in float64 -- the oracle.
  blocked_search                : the device scheme on given scores -- queries in blocks, per (query, slot) candidate
                                  lists of a 128-column tile's two 64-column slots (column quarters p and p + 2), the
                                  strict-greater insert, the merge in tf.nn.top_k's order, then the exclusion.
"""
from __future__ import annotations

import numpy as np

PAD = np.iinfo(np.int32).max
BN = 128            # the wgmma GEMM's N tile


def norms64(table):
    return np.sqrt(np.sum(np.asarray(table, dtype=np.float64) ** 2, axis=1))


def query64(table, ids, weights):
    """sum_w weight_w T_w / |T_w|, scaled to unit length; a zero sum stays zero (gensim's unitvec)."""
    t = np.asarray(table, dtype=np.float64)
    n = norms64(t)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.zeros(t.shape[1])
        for i, w in zip(ids, weights):
            s = s + w * t[i] / n[i]
        ln = np.sqrt(np.sum(s * s))
        return s / ln if ln > 0 else s


def scores64(table, q):
    """s_i = T_i . q / |T_i| in float64; NaN for a zero row."""
    t = np.asarray(table, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return (t @ np.asarray(q, dtype=np.float64)) / norms64(t)


def rank(scores, k):
    """The first k of the rows with a finite score, value descending, ties to the lower row (NaN rows never)."""
    ok = np.flatnonzero(~np.isnan(scores))
    order = ok[np.lexsort((ok, -scores[ok]))]
    return order[:k]


def search64(scores, k, exclude=()):
    """gensim's exclusion: the top k + len(exclude), without the excluded ids, the first k of the rest."""
    best = rank(scores, k + len(exclude))
    ex = set(int(e) for e in exclude)
    return np.array([i for i in best if int(i) not in ex][:k], dtype=np.int64)


def most_similar64(table, word_to_index, positive, negative=(), topn=10):
    ids = [word_to_index[w] for w in list(positive) + list(negative)]
    q = query64(table, ids, [1.0] * len(positive) + [-1.0] * len(negative))
    s = scores64(table, q)
    return [(int(i), float(s[i])) for i in search64(s, topn, ids)], s


def slot_lists(row, kk):
    """The candidate lists of one query's scores: slot 2 t + p of tile t holds the best kk of the columns of quarters p
    and p + 2, inserted in increasing column order with the strict rule x > k-th (ties stay in column order)."""
    N = row.shape[0]
    tiles = (N + BN - 1) // BN
    lists = []
    for t in range(tiles):
        for p in range(2):
            v = [-np.inf] * kk
            i = [PAD] * kk
            for q in (p, p + 2):
                for c in range(t * BN + 32 * q, min(t * BN + 32 * q + 32, N)):
                    x = row[c]
                    if not x > v[-1]:
                        continue
                    at = next(j for j in range(kk) if x > v[j])
                    v.insert(at, x); i.insert(at, c)
                    v.pop(); i.pop()
            lists.append((v, i))
    return lists


def merge(lists, kk):
    """The best kk of the union of sorted lists, tf.nn.top_k's order (value descending, ties to the lower id)."""
    pairs = [(v, i) for vs, ids in lists for v, i in zip(vs, ids) if i != PAD]
    pairs.sort(key=lambda p: (-p[0], p[1]))
    pairs = pairs[:kk]
    return [p[1] for p in pairs] + [PAD] * (kk - len(pairs)), [p[0] for p in pairs] + [-np.inf] * (kk - len(pairs))


def blocked_search(S, k, exclude, block):
    """The device scheme on a score matrix S [nq, N] (float32 scores, as the epilogue forms them): queries in blocks of
    `block`, candidate lists per (query, slot), merge, exclusion.  Returns (ids, values) [nq, k] padded with (PAD, -inf)."""
    nq = S.shape[0]
    kk = k + max((len(e) for e in exclude), default=0)
    ids = np.full((nq, k), PAD, dtype=np.int64)
    vals = np.full((nq, k), -np.inf, dtype=np.float32)
    for r0 in range(0, nq, block):
        for r in range(r0, min(nq, r0 + block)):
            mi, mv = merge(slot_lists(S[r], kk), kk)
            ex = set(exclude[r])
            kept = [(i, v) for i, v in zip(mi, mv) if i == PAD or i not in ex][:k]
            for j, (i, v) in enumerate(kept):
                ids[r, j], vals[r, j] = i, v
    return ids, vals


# ---- error bound of a returned similarity ----------------------------------------------------------------------------
U = 2.0 ** -24
# relative error of one operand as the product reads it: fp32 exact; tf32 drops the 13 low mantissa bits (truncation,
# < 2^-10); 3xTF32 reads hi + lo within 2^-22 of x and drops the lo.lo term (another 2^-22): 2 x 2^-21 per product covers it
OPERAND_EPS = {0: 0.0, 1: 2.0 ** -10, 2: 2.0 ** -21}


def value_bound(mode: int, d: int) -> float:
    """|s_device - s_64| for a unit query: the two operands' rounding (2 eps sum|T_ic q_c| <= 2 eps |T_i| by
    Cauchy-Schwarz, relative to |T_i|), d additions each rounded at most twice (2 d u; tensor-core accumulation is not
    assumed to round to nearest), the query's float32 rounding (u), the float reciprocal norm and the final product
    (2 u), plus slack of 2 u for the norm itself."""
    return 2 * OPERAND_EPS[mode] + (2 * d + 5) * U
