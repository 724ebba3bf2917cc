"""CPU statement of the row-sharded top-k (c2v_topk_partial + c2v_topk_merge): a row's columns are cut into rank blocks
and each block into partial slots; every slot keeps its best k under the strict-greater rule, a rank merges its slots, and
the ranks' lists are merged.  On rows full of exact ties, NaNs and -inf this must give exactly what topk_kernel's rule
gives over the whole row: value descending, ties to the lower index, NaN and -inf never chosen, (-inf, INT_MAX) padding."""
import numpy as np
import pytest

INT_MAX = 2 ** 31 - 1
PAD = (-np.inf, INT_MAX)


def better(a, b):
    """(value, id) a strictly before b: tf.nn.top_k's order (kernels.cuh, better)."""
    return a[0] > b[0] or (a[0] == b[0] and a[1] < b[1])


def strict_list(values, ids, k):
    """A sorted list of k entries fed in increasing id order: an element enters only if strictly greater than the k-th
    value (topk_kernel's per-thread list, EpiTopkT's per-slot list)."""
    lst = [PAD] * k
    for x, j in zip(values, ids):
        if x > lst[-1][0]:
            lst[-1] = (float(x), int(j))
            q = k - 1
            while q > 0 and lst[q][0] > lst[q - 1][0]:
                lst[q], lst[q - 1] = lst[q - 1], lst[q]
                q -= 1
    return lst


def merge(lists, k):
    """topk_merge_kernel: the best k of the union of sorted lists, padding ignored (it sorts last)."""
    out = []
    heads = [0] * len(lists)
    for _ in range(k):
        best, src = PAD, None
        for i, lst in enumerate(lists):
            if heads[i] < len(lst) and better(lst[heads[i]], best):
                best, src = lst[heads[i]], i
        if src is not None:
            heads[src] += 1
        out.append(best)
    return out


def topk_kernel_rule(row, k, threads=256):
    """topk_kernel over a whole row: per-thread strided strict lists, then k rounds of block arg-best over the heads."""
    lists = [strict_list(row[t::threads], np.arange(t, len(row), threads), k) for t in range(threads)]
    return merge(lists, k)


def sharded_topk(row, k, block_edges, slot_len):
    """The scheme: rank blocks [e_r, e_r+1) (global ids), slots of slot_len local columns in each, merged twice."""
    rank_lists = []
    for r0, r1 in zip(block_edges[:-1], block_edges[1:]):
        block = row[r0:r1]
        slots = [strict_list(block[s:s + slot_len], np.arange(s, min(s + slot_len, len(block))) + r0, k)
                 for s in range(0, max(len(block), 1), slot_len)]
        rank_lists.append(merge(slots, k))
    return merge(rank_lists, k)


def nasty_rows(rng, n_rows, Y):
    rows = []
    for i in range(n_rows):
        row = rng.integers(-3, 4, size=Y).astype(np.float32)          # heavy integer ties
        row[rng.random(Y) < 0.1] = np.nan
        row[rng.random(Y) < 0.05] = -np.inf
        if i % 4 == 1:
            row[:] = np.nan                                           # an all-masked bag: every logit NaN
        if i % 4 == 2:
            row[rng.random(Y) < 0.7] = np.nan                         # fewer than k finite values in some blocks
            row[rng.random(Y) < 0.25] = -np.inf
        rows.append(row)
    return rows


@pytest.mark.parametrize("k", [1, 3, 10, 16])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_sharded_scheme_equals_whole_row_rule(k, world):
    rng = np.random.default_rng(1000 * k + world)
    Y = 301
    for row in nasty_rows(rng, 8, Y):
        want = topk_kernel_rule(row, k)
        cuts = np.sort(rng.choice(np.arange(1, Y), size=world - 1, replace=False)) if world > 1 else []
        edges = [0, *[int(c) for c in cuts], Y]
        for slot_len in (1, 5, 64):
            got = sharded_topk(row, k, edges, slot_len)
            assert got == want, (k, world, slot_len, edges, got, want)


def test_contiguous_blocks_smaller_than_k():
    """Y = 37 on 8 ranks in blocks of 5 (the last has 2 rows): blocks pad, the merge ignores the padding."""
    rng = np.random.default_rng(7)
    Y, k, per = 37, 10, 5
    edges = [min(r * per, Y) for r in range(8)] + [Y]
    for row in nasty_rows(rng, 8, Y):
        assert sharded_topk(row, k, edges, 64) == topk_kernel_rule(row, k)


def test_ties_across_a_boundary_resolve_to_the_lower_id():
    row = np.zeros(200, dtype=np.float32)
    row[[37, 99, 100, 150]] = 5.0
    got = sharded_topk(row, 3, [0, 100, 200], 64)
    assert [j for _, j in got] == [37, 99, 100]
    assert got == topk_kernel_rule(row, 3)
