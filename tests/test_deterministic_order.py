"""CPU checks of option "deterministic": the numpy order model, the Trainer's schedule validation and the
C2V_DETERMINISTIC / C2V_SEED parsing (no GPU needed)."""
import numpy as np
import pytest

from tests import deterministic_order as DO


def _naive(rows, vals, n_rows, chunk=DO.K):
    """The documented order written as plain loops."""
    out = np.zeros((n_rows, vals.shape[1]), dtype=np.float32)
    for r in np.unique(rows):
        entries = vals[np.flatnonzero(rows == r)]
        total = np.zeros(vals.shape[1], dtype=np.float32)
        for c0 in range(0, len(entries), chunk):
            acc = np.zeros(vals.shape[1], dtype=np.float32)
            for x in entries[c0:c0 + chunk]:
                acc = acc + x
            total = total + acc
        out[r] = total
    return out


@pytest.mark.parametrize("lengths", [[DO.K - 1], [DO.K], [DO.K + 1], [2 * DO.K + 1], [1, DO.K, 3 * DO.K + 5, 2]])
def test_model_matches_plain_loops_at_chunk_boundaries(lengths):
    rng = np.random.default_rng(len(lengths) * 100 + lengths[0])
    rows = np.concatenate([np.full(n, 3 * i + 1) for i, n in enumerate(lengths)])
    rng.shuffle(rows)
    vals = rng.standard_normal((len(rows), 8)).astype(np.float32) * 10 ** rng.uniform(-3, 3, (len(rows), 1)).astype(np.float32)
    n_rows = 3 * len(lengths) + 2
    got = DO.row_sums(rows, vals, n_rows)
    assert np.array_equal(got.view(np.uint32), _naive(rows, vals, n_rows).view(np.uint32))


def test_model_is_within_the_reordering_bound_of_float64():
    rng = np.random.default_rng(7)
    n_rows = 500
    rows = np.minimum(rng.zipf(1.3, 20000) - 1, n_rows - 1)
    vals = rng.standard_normal((len(rows), 16)).astype(np.float32)
    got = DO.row_sums(rows, vals, n_rows)
    ref = np.zeros((n_rows, 16))
    np.add.at(ref, rows, vals.astype(np.float64))
    assert np.all(np.abs(got - ref) <= DO.reorder_bound(rows, vals, n_rows) + 1e-30)
    untouched = np.bincount(rows, minlength=n_rows) == 0
    assert np.all(got[untouched] == 0)


def test_model_never_produces_negative_zero():
    rows = np.array([0, 0, 1, 1, 1])
    vals = np.array([[-0.0], [-0.0], [1.5], [-1.5], [-0.0]], dtype=np.float32)
    got = DO.row_sums(rows, vals, 2)
    assert not np.signbit(got).any()


def test_trainer_schedule_validation():
    from code2vec_b200.trainer import deterministic_refusal
    for schedule in ("single", "allreduce", "sharded"):
        assert deterministic_refusal(schedule, world=4, push_grads=False) is None
    assert deterministic_refusal("table_sharded", world=1, push_grads=False) is None
    assert deterministic_refusal("fully_sharded", world=1, push_grads=True) is None
    for schedule in ("table_sharded", "fully_sharded"):
        why = deterministic_refusal(schedule, world=2, push_grads=False)
        assert why and "row-sharded" in why
    assert "inbox" in deterministic_refusal("table_sharded", world=8, push_grads=True)


def test_seed_and_mode_parsing():
    from code2vec_b200.b200_model import DEFAULT_DETERMINISTIC_SEED, run_determinism
    assert run_determinism({"C2V_DETERMINISTIC": "1"}) == (True, DEFAULT_DETERMINISTIC_SEED)
    assert run_determinism({"C2V_DETERMINISTIC": "1", "C2V_SEED": "7"}) == (True, 7)
    assert run_determinism({"C2V_SEED": "8"}) == (False, 8)
    det, seed = run_determinism({}, now=lambda: 1234.5)
    assert det is False and seed == 1234
    det, seed = run_determinism({"C2V_DETERMINISTIC": "0"}, now=lambda: 2.0 ** 40 + 3)
    assert det is False and 0 <= seed <= 0x7FFFFFFF
    for bad in ({"C2V_DETERMINISTIC": "yes"}, {"C2V_SEED": "x"}, {"C2V_SEED": "-1"}):
        with pytest.raises(ValueError):
            run_determinism(bad)
