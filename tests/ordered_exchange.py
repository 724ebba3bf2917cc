"""numpy model of option "ordered_exchange" (include/c2v_b200.h, DESIGN.md section 5.1): the gradient of a row of a table
that is row-sharded over W ranks (global row r on rank r % W, local row r // W).

Sender s reduces its own contributions to the row to one sum R_s in the order of option "deterministic"
(tests/deterministic_order.row_sums: entries in list order, chunks of 32 from the row's first entry, each summed left to
right from +0.0, chunk sums added left to right from +0.0).  The owner stores G, where G = +0.0 and then G = fl(G + R_s)
for s = 0, 1, ..., W - 1, skipping the senders that have no entry for the row.  Rows nobody references are not written."""
import numpy as np

from tests import deterministic_order as DO


def fold(senders, n_rows, sender_order=None):
    """senders[s] = (rows, vals): global row ids [n] and float32 contributions [n, d] of sender s, in entry order.
    Returns (G [n_rows, d] float32, referenced [n_rows] bool); G is meaningful where referenced.  sender_order: the order
    in which the owner adds the senders' sums (default 0 .. W-1, which is the specification)."""
    d = np.asarray(senders[0][1]).shape[1]
    G = np.zeros((n_rows, d), dtype=np.float32)
    referenced = np.zeros(n_rows, dtype=bool)
    for s in (range(len(senders)) if sender_order is None else sender_order):
        rows = np.asarray(senders[s][0], dtype=np.int64)
        if rows.size == 0:
            continue
        R = DO.row_sums(rows, senders[s][1], n_rows)
        has = np.bincount(rows, minlength=n_rows) > 0
        G[has] = G[has] + R[has]                  # one float32 addition per element
        referenced |= has
    return G, referenced


def shard(table, owner, world):
    """Rows of a global table that rank `owner` holds, in local-row order."""
    return table[owner::world]


def pushed_records(src, pth, tgt, mask):
    """(row, sum) records one sender pushes for a batch: its distinct unmasked token rows (source and target columns) plus
    its distinct unmasked path rows."""
    live = np.asarray(mask) != 0
    tok = np.union1d(np.asarray(src)[live], np.asarray(tgt)[live])
    return int(tok.size + np.unique(np.asarray(pth)[live]).size)
