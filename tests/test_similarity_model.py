"""CPU checks of the nearest-neighbour search (DESIGN.md §6h): the float64 oracle against gensim's definition, the numpy
model of the device's block / slot / merge / exclusion scheme against the oracle at tile, slot and block edges, and the
command line's parsing and output formats."""
import io

import numpy as np
import pytest

from code2vec_b200 import similarity as S
from code2vec_b200.__main__ import print_most_similar
from tests import similarity_model as M


def _table(n, d, seed):
    return np.random.default_rng(seed).standard_normal((n, d)).astype(np.float32)


def test_oracle_states_gensim_most_similar():
    t = _table(50, 8, 1)
    w2i = {"w%d" % i: i for i in range(50)}
    got, s = M.most_similar64(t, w2i, ["w3", "w7"], ["w9"], topn=5)
    n = t / np.linalg.norm(t.astype(np.float64), axis=1, keepdims=True)
    mean = n[3] + n[7] - n[9]
    mean = mean / np.linalg.norm(mean)
    dist = n @ mean
    order = [i for i in np.argsort(-dist, kind="stable")[:8] if i not in (3, 7, 9)][:5]
    assert [i for i, _ in got] == order
    assert np.allclose([v for _, v in got], dist[order], rtol=0, atol=1e-12)


def test_oracle_edges():
    t = _table(10, 4, 2)
    t[4] = 0.0                                        # zero row: NaN, never returned
    q = M.query64(t, [1, 1], [1.0, -1.0])             # p = n: a zero query, every finite score 0: ids ascending
    assert not q.any()
    s = M.scores64(t, q)
    assert np.isnan(s[4])
    assert list(M.search64(s, 20, [1, 1])) == [0, 2, 3, 5, 6, 7, 8, 9]   # fewer than k rows remain: fewer returned


def _check_model(S32, k, exclude, block):
    ids, vals = M.blocked_search(S32, k, exclude, block)
    for r in range(S32.shape[0]):
        want = M.search64(S32[r].astype(np.float64), k, exclude[r])
        got = [i for i in ids[r] if i != M.PAD]
        assert got == list(want), r
        assert np.array_equal(vals[r, :len(got)], S32[r, want])


@pytest.mark.parametrize("N", [1, 37, 63, 64, 65, 127, 128, 129, 300])
@pytest.mark.parametrize("k", [1, 10, 16])
def test_scheme_matches_oracle_at_tile_and_slot_edges(N, k):
    rng = np.random.default_rng(N * 100 + k)
    nq = 5
    S32 = rng.standard_normal((nq, N)).astype(np.float32)
    S32[:, ::7] = np.float32(0.5)                     # exact ties across slots and tiles
    if N > 3:
        S32[:, 3] = np.nan                            # a zero row
    exclude = [list(rng.integers(0, N, size=int(rng.integers(0, 3)))) for _ in range(nq)]
    exclude[0] = [0, 0]                               # a duplicated word counts twice
    _check_model(S32, k, exclude, block=2)


def test_scheme_ties_across_slot_tile_and_block_edges():
    N = 300
    S32 = np.full((7, N), -1.0, dtype=np.float32)
    for c in (31, 32, 63, 64, 127, 128, 129, 255, 256):  # quarter, slot and tile boundaries
        S32[:, c] = 0.75
    exclude = [[] for _ in range(7)]
    exclude[3] = [64]
    ids, _ = M.blocked_search(S32, 9, exclude, block=3)
    assert list(ids[0]) == [31, 32, 63, 64, 127, 128, 129, 255, 256]
    assert list(ids[3][:8]) == [31, 32, 63, 127, 128, 129, 255, 256]
    _check_model(S32, 9, exclude, block=3)


def test_value_bound_is_derived_from_the_modes():
    assert M.value_bound(0, 128) < M.value_bound(2, 128) < M.value_bound(1, 128)
    assert M.value_bound(1, 384) < 3e-3 and M.value_bound(0, 384) < 1e-4


def test_query_lines():
    assert S.parse_query_line("equals,to|lower\n") == (["equals", "to|lower"], [])
    assert S.parse_query_line("download,send receive") == (["download", "send"], ["receive"])
    assert S.parse_query_line("   \n") is None
    with pytest.raises(ValueError):
        S.parse_query_line("a b c")


def test_cli_flags_are_removed_from_argv():
    argv, a = S.split_cli_flags(["--load", "m", "--most_similar", "token", "--topn", "3", "--most_similar_input", "q.txt",
                                 "--nearest", "c.c2v"])
    assert argv == ["--load", "m"]
    assert (a.most_similar, a.topn, a.most_similar_input, a.nearest) == ("token", 3, "q.txt", "c.c2v")
    argv, a = S.split_cli_flags(["--load", "m"])
    assert argv == ["--load", "m"] and not a.active and a.topn == 10


@pytest.mark.parametrize("argv", [["--most_similar"], ["--nearest"], ["--topn", "--load"], ["--most_similar", "words"],
                                  ["--topn", "0"], ["--topn", "x"]])
def test_cli_flag_errors(argv):
    with pytest.raises(ValueError):
        S.split_cli_flags(argv)


def test_more_than_one_gpu_is_refused_before_any_work():
    _, a = S.split_cli_flags(["--nearest", "c.c2v"])
    with pytest.raises(ValueError):
        S.check_single_gpu(a, 2)
    S.check_single_gpu(a, 1)
    S.check_single_gpu(S.SimilarityArgs(), 4)


def test_main_refuses_several_ranks(monkeypatch):
    from code2vec_b200 import __main__ as main_mod
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(ValueError, match="one GPU"):
        main_mod.main(["--load", "nowhere", "--most_similar", "target"])


def test_output_formats():
    assert S.format_most_similar("a,b c\n", [("x", 0.5), ("y", -0.25)]) == \
        "Most similar to:\ta,b c\n\t(0.500000) x\n\t(-0.250000) y\n"
    assert S.format_nearest_line("get|name", [(4, "set|name", 0.875), (0, "get|id", 0.5)]) == \
        "get|name\t4,set|name,0.875000\t0,get|id,0.500000\n"


class _FakeVocab:
    word_to_index = {"a": 0, "b": 1}


class _FakeModel:
    class vocabs:
        @staticmethod
        def get(_):
            return _FakeVocab

    def most_similar(self, positive, negative, topn, vocab_type):
        return [("b", 1.0)][:topn]


def test_unknown_words_are_reported_and_the_run_moves_on():
    out = io.StringIO()
    print_most_similar(_FakeModel(), None, ["a zz\n", "\n", "a\n"], 1, out)
    assert out.getvalue() == "Not in vocabulary: zz\nMost similar to:\ta\n\t(1.000000) b\n"
