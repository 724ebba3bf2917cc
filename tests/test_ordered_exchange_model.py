"""The numpy statement of option "ordered_exchange" (tests/ordered_exchange.py): what it equals, what it is invariant to,
what it depends on -- so that the GPU comparison against it (tests/test_gpu_ordered_exchange.py) means something."""
import numpy as np

from tests import deterministic_order as DO
from tests import ordered_exchange as OX


def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def _vals(rng, n, d=8):
    return (rng.standard_normal((n, d)) * 2.0 ** rng.uniform(-20, 20, (n, 1))).astype(np.float32)


def test_one_sender_is_the_deterministic_row_sum():
    rng = np.random.default_rng(1)
    rows = rng.integers(0, 40, 3000)
    rows[:1100] = 7                                    # more than 32 chunks
    vals = _vals(rng, len(rows))
    G, ref = OX.fold([(rows, vals)], 50)
    want = DO.row_sums(rows, vals, 50)
    assert np.array_equal(ref, np.bincount(rows, minlength=50) > 0)
    assert np.array_equal(_bits(G[ref]), _bits((np.float32(0.0) + want)[ref]))
    assert not G[~ref].any()
    # two senders with disjoint rows: every row is its only sender's sum
    lo = rows < 20
    G2, _ = OX.fold([(rows[lo], vals[lo]), (rows[~lo], vals[~lo])], 50)
    assert np.array_equal(_bits(G2), _bits(G))


def test_invariant_to_how_different_rows_interleave():
    rng = np.random.default_rng(2)
    senders = []
    for s in range(4):
        rows = rng.integers(0, 30, 2000)
        senders.append((rows, _vals(rng, len(rows))))
    G, ref = OX.fold(senders, 30)
    shuffled = []
    for rows, vals in senders:                         # stable regrouping by row: each row keeps its own entry order
        order = np.argsort(rng.permutation(30)[rows], kind="stable")
        assert not np.array_equal(order, np.arange(len(rows)))
        shuffled.append((rows[order], vals[order]))
    G2, ref2 = OX.fold(shuffled, 30)
    assert np.array_equal(ref, ref2) and np.array_equal(_bits(G), _bits(G2))


def test_depends_on_the_sender_order():
    # row 3: senders 0, 1, 2 hold 2^20, -2^20, 2^-20.  In rank order the big terms cancel first and 2^-20 survives; in the
    # reverse order 2^-20 is absorbed by -2^20
    one = lambda x: (np.array([3]), np.full((1, 4), x, dtype=np.float32))
    senders = [one(2.0 ** 20), one(-2.0 ** 20), one(2.0 ** -20)]
    G, _ = OX.fold(senders, 5)
    Gr, _ = OX.fold(senders, 5, sender_order=[2, 1, 0])
    assert np.all(G[3] == np.float32(2.0 ** -20)) and np.all(Gr[3] == 0.0)
    # and on the entry order inside one sender
    rows = np.array([3, 3, 3])
    vals = np.array([[2.0 ** 20], [-2.0 ** 20], [2.0 ** -20]], dtype=np.float32).repeat(4, axis=1)
    a, _ = OX.fold([(rows, vals)], 5)
    b, _ = OX.fold([(rows, vals[::-1])], 5)
    assert not np.array_equal(_bits(a), _bits(b))


def test_never_yields_negative_zero():
    nz = np.full((1, 4), -0.0, dtype=np.float32)
    cases = [[(np.array([1]), nz)],
             [(np.array([1]), nz), (np.array([1]), nz)],
             [(np.array([1, 1]), np.concatenate([nz, nz])), (np.zeros(0, dtype=np.int64), np.zeros((0, 4), np.float32))],
             [(np.array([1]), np.full((1, 4), 1.5, np.float32)), (np.array([1]), np.full((1, 4), -1.5, np.float32))]]
    for senders in cases:
        G, ref = OX.fold(senders, 3)
        assert ref[1] and not np.signbit(G).any() and not G.any()


def test_shards_and_record_counts():
    table = np.arange(11)[:, None]
    assert [OX.shard(table, o, 4)[:, 0].tolist() for o in range(4)] == [[0, 4, 8], [1, 5, 9], [2, 6, 10], [3, 7]]
    src = np.array([[1, 2, 9], [1, 1, 9]])
    tgt = np.array([[2, 3, 9], [4, 1, 9]])
    pth = np.array([[5, 5, 9], [6, 5, 9]])
    mask = np.array([[1, 1, 0], [1, 1, 0]], dtype=np.float32)
    assert OX.pushed_records(src, pth, tgt, mask) == 4 + 2        # tokens {1, 2, 3, 4}, paths {5, 6}; 9 is masked


def test_deterministic_refusal_with_ordered_exchange():
    from code2vec_b200.trainer import deterministic_refusal
    for schedule in ("table_sharded", "fully_sharded"):
        for world in (2, 4, 8):
            for push in (False, True):
                assert deterministic_refusal(schedule, world, push, ordered_exchange=True) is None
                assert deterministic_refusal(schedule, world, push, ordered_exchange=False) == \
                    deterministic_refusal(schedule, world, push)
                assert deterministic_refusal(schedule, world, push)
    for schedule in ("single", "allreduce", "sharded"):
        assert deterministic_refusal(schedule, 4, False, ordered_exchange=True) is None
