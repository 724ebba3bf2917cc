"""CPU checks of the name scores (DESIGN.md §6n): the float64 statement's rank rule (tests/name_scores_model.py) against a
brute-force sort in tf.nn.top_k's order, and the host side of `--score_names` (code2vec_b200/name_scores.py)."""
import math

import numpy as np
import pytest

from code2vec_b200 import name_scores as N
from tests.name_scores_model import name_scores64


def _sorted_rank(row, y):
    """1-based position of y when the row is sorted value descending, exact ties to the lower index."""
    cols = np.arange(row.size)
    order = np.lexsort((cols, -np.asarray(row, dtype=np.float64)))
    return int(np.flatnonzero(order == y)[0]) + 1


def _check_against_sort(S, y):
    rank, logp, top1, top1_logp = name_scores64(S, y)
    for b in range(S.shape[0]):
        assert rank[b] == _sorted_rank(S[b], y[b]), b
        assert _sorted_rank(S[b], top1[b]) == 1
        p = np.exp(S[b].astype(np.float64) - S[b].max())
        assert math.isclose(logp[b], math.log(p[y[b]] / p.sum()), rel_tol=1e-12, abs_tol=1e-12)
        assert math.isclose(top1_logp[b], math.log(1.0 / p.sum()), rel_tol=1e-12, abs_tol=1e-12)
        assert (rank[b] == 1) == (top1[b] == y[b])


def test_random_rows():
    rng = np.random.default_rng(1)
    for Y in (2, 3, 127, 128, 129, 1000):
        S = rng.standard_normal((9, Y)).astype(np.float32)
        _check_against_sort(S, rng.integers(0, Y, size=9))


def test_exact_ties_at_above_and_below_the_target():
    rng = np.random.default_rng(2)
    Y = 64
    S = rng.integers(-3, 4, size=(40, Y)).astype(np.float32)     # few distinct values: ties everywhere
    y = rng.integers(0, Y, size=40)
    _check_against_sort(S, y)
    row = np.array([1, 5, 3, 5, 3, 0, 3, 5], dtype=np.float32)
    r, _, t1, _ = name_scores64(np.stack([row] * 4), [2, 4, 6, 3])
    assert r.tolist() == [4, 5, 6, 2]          # the 5s (1, 3, 7) first, then the 3s (2, 4, 6) in index order
    assert t1.tolist() == [1, 1, 1, 1]


def test_signed_zeros_are_equal():
    row = np.array([-0.0, 0.0, -0.0, -1.0, 0.0], dtype=np.float32)
    S = np.stack([row] * 5)
    y = np.arange(5)
    rank, logp, top1, _ = name_scores64(S, y)
    assert rank.tolist() == [1, 2, 3, 5, 4]
    assert top1.tolist() == [0] * 5
    _check_against_sort(S, y)


def test_nan_row_is_never_ranked():
    S = np.array([[0.5, np.nan, 2.0, 2.0], [0.5, 1.0, 2.0, 3.0]], dtype=np.float32)
    rank, logp, top1, top1_logp = name_scores64(S, [0, 0])
    assert rank[0] == 0 and np.isnan(logp[0]) and np.isnan(top1_logp[0])
    assert top1[0] == 2                        # the first of the largest non-NaN logits
    assert rank[1] == 4 and top1[1] == 3


def test_one_target_row():
    rank, logp, top1, top1_logp = name_scores64(np.array([[3.5], [-2.0]], dtype=np.float32), [0, 0])
    assert rank.tolist() == [1, 1] and top1.tolist() == [0, 0]
    assert logp.tolist() == [0.0, 0.0] and top1_logp.tolist() == [0.0, 0.0]


# ---- the command line ---------------------------------------------------------------------------------------------------
def test_flag_split():
    argv, path = N.split_cli_flags(["--load", "m", "--score_names", "a.c2v", "--framework", "b200"])
    assert argv == ["--load", "m", "--framework", "b200"] and path == "a.c2v"
    assert N.split_cli_flags(["--load", "m"]) == (["--load", "m"], None)
    for bad in (["--load", "m", "--score_names"], ["--score_names", "--load", "m"]):
        with pytest.raises(ValueError, match="needs an argument"):
            N.split_cli_flags(bad)
    with pytest.raises(ValueError, match="given 2 times"):
        N.split_cli_flags(["--score_names", "a.c2v", "--score_names", "b.c2v"])


def test_several_ranks_are_refused_before_any_engine_exists(monkeypatch):
    from code2vec_b200 import __main__ as main_mod
    N.check_single_gpu("a.c2v", 1)
    N.check_single_gpu(None, 8)
    with pytest.raises(ValueError, match="one GPU"):
        N.check_single_gpu("a.c2v", 2)

    def no_model(_config):
        raise AssertionError("a model was built")
    monkeypatch.setattr(main_mod, "load_model_dynamically", no_model)
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(ValueError, match="--score_names runs on one GPU; this run has 2 ranks"):
        main_mod.main(["--load", "nowhere", "--score_names", "a.c2v"])


def test_line_format():
    assert N.format_line("get|name", True, 3, -1.25, "set|name", -0.5) == "get|name\t3\t-1.250000\tset|name\t-0.500000\n"
    assert N.format_line("no|such", False, 7, -9.0, "get|id", -0.125) == "no|such\t-\t-\tget|id\t-0.125000\n"
    assert N.format_line("x", True, 0, float("nan"), "y", float("nan")) == "x\t-\tnan\ty\tnan\n"


def test_summary():
    rank = np.array([1, 4, 2, 9, 1], dtype=np.int32)
    logp = np.array([-0.5, -2.0, -1.0, -7.0, -0.25], dtype=np.float32)
    in_vocab = np.array([True, True, True, False, True])
    n, n_in, mean_logp, mrr = N.summarize(rank, logp, in_vocab)
    assert (n, n_in) == (5, 4)
    assert mean_logp == pytest.approx((-0.5 - 2.0 - 1.0 - 0.25) / 4, abs=1e-15)
    assert mrr == pytest.approx((1 + 0.25 + 0.5 + 1) / 4, abs=1e-15)
    line = N.summary_line(rank, logp, in_vocab)
    assert line == ("Name scores: 5 rows, 4 with in-vocabulary names; over those, mean log p(name) = -0.937500, "
                    "mean reciprocal rank = 0.687500")
    n, n_in, mean_logp, mrr = N.summarize([0, 2], [float("nan"), -1.0], [True, True])
    assert math.isnan(mean_logp) and mrr == 0.25
    n, n_in, mean_logp, mrr = N.summarize([3], [-1.0], [False])
    assert (n, n_in) == (1, 0) and math.isnan(mean_logp) and math.isnan(mrr)
