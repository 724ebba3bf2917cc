"""numpy model of the summation order of option "deterministic" (include/c2v_b200.h, DESIGN.md section 5.1).

A gradient row's contributions, listed in increasing entry order, are cut into chunks of K entries starting at the row's
first entry; each chunk is summed left to right in float32 from +0.0, and the chunk sums are added left to right from
+0.0.  The engine's sort + chunked reduce (c2v_selftest_row_sum) must reproduce this bit for bit."""
import numpy as np

K = 32          # kDetChunk in csrc/kernels.cuh


def row_sums(rows, vals, n_rows, chunk=K):
    """Table [n_rows, d] (float32, zero where no entry) in which row r holds the ordered chunked sum of vals[i] over the
    entries i (in increasing i) with rows[i] == r.  Vectorised over chunks: step k adds the k-th entry of every chunk
    that has one, so each chunk still sees its entries left to right."""
    rows = np.asarray(rows, dtype=np.int64)
    vals = np.asarray(vals, dtype=np.float32)
    d = vals.shape[1]
    out = np.zeros((n_rows, d), dtype=np.float32)
    if rows.size == 0:
        return out
    order = np.argsort(rows, kind="stable")
    srows = rows[order]
    head = np.ones(len(srows), dtype=bool)
    head[1:] = srows[1:] != srows[:-1]
    seg_start = np.maximum.accumulate(np.where(head, np.arange(len(srows)), 0))
    pos = np.arange(len(srows)) - seg_start
    off, chunk_of_row = pos % chunk, pos // chunk
    cid = np.cumsum(off == 0) - 1                           # global chunk id of every sorted entry
    sums = np.zeros((int(cid[-1]) + 1, d), dtype=np.float32)
    for k in range(chunk):
        sel = off == k
        sums[cid[sel]] += vals[order[sel]]                  # one entry per chunk: a plain float32 addition each
    first = off == 0
    c_row, c_j = srows[first], chunk_of_row[first]
    for j in range(int(c_j.max()) + 1):
        sel = c_j == j
        out[c_row[sel]] += sums[sel]                        # chunk j of every row that has one, rows distinct
    return out


def reorder_bound(rows, vals, n_rows):
    """Per-element bound on |sum in any fp32 order - exact sum|: n * eps32 * sum |v| (n = entries of the row)."""
    rows = np.asarray(rows, dtype=np.int64)
    absum = np.zeros((n_rows, np.asarray(vals).shape[1]), dtype=np.float64)
    np.add.at(absum, rows, np.abs(np.asarray(vals, dtype=np.float64)))
    cnt = np.bincount(rows, minlength=n_rows).astype(np.float64)[:, None]
    return cnt * np.finfo(np.float32).eps * absum
