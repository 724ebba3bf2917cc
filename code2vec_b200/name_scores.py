"""Each method's own name scored over the whole target vocabulary (DESIGN.md §6n): the host side of
`python -m code2vec_b200 --load M --score_names FILE.c2v`.

For every example evaluate() would score in FILE.c2v, `Code2VecModel.score_names` runs the engine's c2v_name_scores on the
GPU: the full-softmax log-probability of the method's actual name, its 1-based rank among all target names in
tf.nn.top_k's order, and the model's top-1 name with its log-probability.  This module holds what needs no GPU: the flag,
the line format of FILE.c2v.name_scores and the summary line.

    name<TAB>rank<TAB>logp<TAB>top1_name<TAB>top1_logp

A name outside the target vocabulary prints `-` for its rank and logp (it is scored as the target OOV word, which is not
the name); a row whose logits hold a NaN has rank 0, printed `-`, and `nan` log-probabilities."""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import numpy as np

FLAG = "--score_names"
SUFFIX = ".name_scores"


def split_cli_flags(argv: Sequence[str]) -> Tuple[List[str], Optional[str]]:
    """argv without `--score_names FILE`, and FILE (None without the flag).  ValueError for the flag without a value or
    given twice."""
    argv = list(argv)
    if argv.count(FLAG) > 1:
        raise ValueError("%s is given %d times; score one file per run" % (FLAG, argv.count(FLAG)))
    if FLAG not in argv:
        return argv, None
    i = argv.index(FLAG)
    if i + 1 >= len(argv) or argv[i + 1].startswith("--"):
        raise ValueError("%s needs an argument" % FLAG)
    path = argv[i + 1]
    del argv[i:i + 2]
    return argv, path


def check_single_gpu(path: Optional[str], world: int):
    """--score_names runs on one GPU, as --nearest does: on several ranks each holds only a block of the target table."""
    if path is not None and world > 1:
        raise ValueError("--score_names runs on one GPU; this run has %d ranks" % world)


def format_line(name: str, in_vocab: bool, rank: int, logp: float, top1_name: str, top1_logp: float) -> str:
    """One line of FILE.c2v.name_scores: `-` for the rank and logp of a name outside the target vocabulary, and for the
    rank 0 of a row whose logits hold a NaN."""
    r = "%d" % rank if in_vocab and rank > 0 else "-"
    lp = "%.6f" % logp if in_vocab else "-"
    return "%s\t%s\t%s\t%s\t%.6f\n" % (name, r, lp, top1_name, top1_logp)


def summarize(rank, logp, in_vocab) -> Tuple[int, int, float, float]:
    """(rows, rows with an in-vocabulary name, mean logp and mean reciprocal rank over those), in float64.  A row with
    NaN logits (rank 0) counts 0 towards the MRR and makes the mean logp NaN.  Both means are NaN without such rows."""
    rank = np.asarray(rank, dtype=np.int64)
    logp = np.asarray(logp, dtype=np.float64)
    keep = np.asarray(in_vocab, dtype=bool)
    n_in = int(keep.sum())
    if n_in == 0:
        return int(rank.size), 0, math.nan, math.nan
    r = rank[keep]
    rr = np.where(r > 0, 1.0 / np.maximum(r, 1), 0.0)
    return int(rank.size), n_in, float(logp[keep].mean()), float(rr.mean())


def summary_line(rank, logp, in_vocab) -> str:
    n, n_in, mean_logp, mrr = summarize(rank, logp, in_vocab)
    return ("Name scores: %d rows, %d with in-vocabulary names; over those, mean log p(name) = %.6f, mean reciprocal "
            "rank = %.6f" % (n, n_in, mean_logp, mrr))
