"""Nearest-neighbour search on the GPU (DESIGN.md §6h): gensim's `KeyedVectors.most_similar` over the trained embedding
tables, and the nearest methods of a corpus by code vector.

The reference README tells users to export the tables as word2vec text and query them with gensim:

    model.most_similar(positive=['equals', 'to|lower'])
    model.most_similar(positive=['download', 'send'], negative=['receive'])

Here the same query runs against the table in device memory (c2v_knn_*, include/c2v_b200.h "Nearest neighbours"):
  * query : the sum of +T_w / |T_w| over the positive words and -T_w / |T_w| over the negative ones, scaled to unit
            length (a zero sum stays zero);
  * score : s_i = (T_i . q) / |T_i|; a row of zero norm scores NaN and is never returned;
  * result: the top topn + len(words), without the query's words (a repeated word counts twice), the first topn of
            the rest; value descending, exact ties to the lower row.  An unknown word raises KeyError as gensim does.
The command line (`python -m code2vec_b200`) adds `--most_similar {target,token,path}` with `--most_similar_input FILE`,
`--nearest CORPUS.c2v` and `--topn N`; split_cli_flags takes them out of argv so that Config stays the reference's."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np

from .engine import EngineError, load_library

MAX_CANDIDATES = 64          # k + excluded words the search accepts at all
TABLES = ("target", "token", "path")


# ---- command line --------------------------------------------------------------------------------------------------
@dataclass
class SimilarityArgs:
    most_similar: Optional[str] = None        # "target", "token" or "path"
    most_similar_input: Optional[str] = None  # queries file; None = standard input
    nearest: Optional[str] = None             # a `.c2v` corpus
    topn: int = 10

    @property
    def active(self) -> bool:
        return self.most_similar is not None or self.nearest is not None


def split_cli_flags(argv: Sequence[str]) -> Tuple[List[str], SimilarityArgs]:
    """argv without --most_similar, --most_similar_input, --nearest and --topn (each followed by its value), and their
    values.  ValueError for a flag without a value, an unknown table or topn < 1."""
    argv = list(argv)
    out = SimilarityArgs()
    for flag in ("--most_similar", "--most_similar_input", "--nearest", "--topn"):
        while flag in argv:
            i = argv.index(flag)
            if i + 1 >= len(argv) or argv[i + 1].startswith("--"):
                raise ValueError("%s needs an argument" % flag)
            value = argv[i + 1]
            del argv[i:i + 2]
            if flag == "--most_similar":
                if value not in TABLES:
                    raise ValueError("--most_similar takes one of %s, got %r" % (", ".join(TABLES), value))
                out.most_similar = value
            elif flag == "--most_similar_input":
                out.most_similar_input = value
            elif flag == "--nearest":
                out.nearest = value
            else:
                try:
                    out.topn = int(value)
                except ValueError:
                    raise ValueError("--topn needs an integer, got %r" % value) from None
                if out.topn < 1:
                    raise ValueError("--topn must be at least 1, got %d" % out.topn)
    return argv, out


def check_single_gpu(args: SimilarityArgs, world: int):
    """--most_similar and --nearest run on one GPU, as --predict and --release do."""
    if args.active and world > 1:
        raise ValueError("--most_similar and --nearest run on one GPU; this run has %d ranks" % world)


def parse_query_line(line: str) -> Optional[Tuple[List[str], List[str]]]:
    """`pos1,pos2[ neg1,neg2]` -> (positive words, negative words); None for a blank line.  Words never hold spaces or
    commas: `.c2v` fields are split on them."""
    fields = line.strip().split()
    if not fields:
        return None
    if len(fields) > 2:
        raise ValueError("a query is `positive,words [negative,words]`, got %r" % line.strip())
    words = [[w for w in f.split(",") if w] for f in fields]
    return words[0], (words[1] if len(words) > 1 else [])


def format_most_similar(line: str, results: Sequence[Tuple[str, float]]) -> str:
    return "Most similar to:\t%s\n" % line.strip() + "".join("\t(%f) %s\n" % (v, w) for w, v in results)


def format_nearest_line(name: str, neighbours: Sequence[Tuple[int, str, float]]) -> str:
    """One line of `<corpus>.nearest`: the example's name, then `\\t<row>,<name>,<similarity>` per neighbour."""
    return name + "".join("\t%d,%s,%f" % (r, n, v) for r, n, v in neighbours) + "\n"


# ---- the native search -----------------------------------------------------------------------------------------------
class NearestNeighbours:
    """A c2v_knn handle on `device`: bind a float32 table [N, d] in device memory, build gensim's query vectors, search.
    The bound tensor is kept alive; bind again after its contents change."""

    def __init__(self, device):
        import torch
        self.torch = torch
        self.lib = load_library()
        self.dev = torch.device(device)
        self.h = C.c_void_p()
        self._check(self.lib.c2v_knn_create(self.dev.index or 0, C.byref(self.h)))
        self.table = None
        self.math = None

    def _check(self, rc: int):
        if rc != 0:
            raise EngineError(rc, self.lib.c2v_last_error(None).decode())

    def _stream(self):
        return self.torch.cuda.current_stream(self.dev).cuda_stream

    def bind(self, table, math: int):
        torch = self.torch
        if table.dim() != 2 or table.dtype != torch.float32 or table.device != self.dev or table.stride(1) != 1:
            raise ValueError("bind needs a row-major 2-d float32 tensor on %s" % self.dev)
        self._check(self.lib.c2v_knn_bind_table(self.h, table.data_ptr(), int(table.shape[0]), int(table.shape[1]),
                                                int(table.stride(0)), int(math), self._stream()))
        self.table, self.math = table, int(math)

    def queries(self, ids, weights, offsets):
        """[nq, d] query vectors: query j from the row ids ids[offsets[j]:offsets[j + 1]] with those weights."""
        torch = self.torch
        n_rows = int(self.table.shape[0])
        ids = np.asarray(ids, dtype=np.int64)
        if ids.size and (ids.min() < 0 or ids.max() >= n_rows):
            raise IndexError("query word ids must be in [0, %d)" % n_rows)
        offsets = np.asarray(offsets, dtype=np.int64)
        nq = int(offsets.size) - 1
        d_ids = torch.from_numpy(ids.astype(np.int32)).to(self.dev)
        d_w = torch.from_numpy(np.asarray(weights, dtype=np.float32)).to(self.dev)
        d_off = torch.from_numpy(offsets).to(self.dev)
        q = torch.empty((nq, int(self.table.shape[1])), dtype=torch.float32, device=self.dev)
        self._check(self.lib.c2v_knn_queries(self.h, d_ids.data_ptr(), d_w.data_ptr(), d_off.data_ptr(), nq,
                                             q.data_ptr(), self._stream()))
        return q

    def search(self, q, k: int, exclude: Optional[Sequence[Sequence[int]]] = None, exclude_self: bool = False):
        """(ids [nq, k] int32, values [nq, k] float32) device tensors for the queries q [nq, d]: the best k rows of each
        after dropping its excluded ids -- exclude[j] (a list per query), or with exclude_self the id j itself --
        padded with (INT_MAX, -inf)."""
        torch = self.torch
        nq = int(q.shape[0])
        if q.stride(1) != 1:
            q = q.contiguous()
        x = x_off = None
        max_ex = 0
        if exclude_self:
            x = torch.arange(nq, dtype=torch.int32, device=self.dev)
            x_off = torch.arange(nq + 1, dtype=torch.int64, device=self.dev)
            max_ex = 1
        elif exclude is not None:
            lens = [len(e) for e in exclude]
            max_ex = max(lens, default=0)
            off = np.zeros(nq + 1, dtype=np.int64)
            np.cumsum(lens, out=off[1:])
            flat = np.concatenate([np.asarray(e, dtype=np.int32) for e in exclude] + [np.zeros(1, np.int32)])
            x = torch.from_numpy(flat).to(self.dev)
            x_off = torch.from_numpy(off).to(self.dev)
        idx = torch.empty((nq, k), dtype=torch.int32, device=self.dev)
        val = torch.empty((nq, k), dtype=torch.float32, device=self.dev)
        self._check(self.lib.c2v_knn_search(self.h, q.data_ptr(), nq, int(q.stride(0)), int(k),
                                            None if x is None else x.data_ptr(), None if x_off is None else x_off.data_ptr(),
                                            max_ex, idx.data_ptr(), val.data_ptr(), self._stream()))
        return idx, val

    def profile(self, on: bool) -> Tuple[float, float]:
        """(GEMM ms, selection ms) of the searches since the last call; on: time the searches that follow."""
        g, s = C.c_double(), C.c_double()
        self._check(self.lib.c2v_knn_profile(self.h, int(on), C.byref(g), C.byref(s)))
        return g.value, s.value

    def device_bytes(self) -> int:
        return int(self.lib.c2v_knn_device_bytes(self.h))

    def close(self):
        if self.h:
            self.lib.c2v_knn_destroy(self.h)
            self.h = C.c_void_p()
        self.table = None


def most_similar(nn: NearestNeighbours, word_to_index, index_to_word, positive: Iterable[str],
                 negative: Iterable[str] = (), topn: int = 10) -> List[Tuple[str, float]]:
    """gensim 4's KeyedVectors.most_similar(positive, negative, topn) on the table bound to nn."""
    positive, negative = list(positive), list(negative)
    if topn < 1:
        return []
    ids = []
    for w in positive + negative:
        if w not in word_to_index:
            raise KeyError("Key '%s' not present in vocabulary" % w)
        ids.append(int(word_to_index[w]))
    if not ids:
        raise ValueError("cannot compute similarity with no input")
    if topn + len(ids) > MAX_CANDIDATES:
        raise ValueError("topn + the number of query words may be at most %d" % MAX_CANDIDATES)
    q = nn.queries(ids, [1.0] * len(positive) + [-1.0] * len(negative), [0, len(ids)])
    idx, val = nn.search(q, topn, exclude=[ids])
    idx, val = idx[0].cpu().numpy(), val[0].cpu().numpy()
    return [(index_to_word[int(i)], float(v)) for i, v in zip(idx, val) if i != np.iinfo(np.int32).max]


def nearest_rows_device(nn: NearestNeighbours, vectors, topn: int, math: int):
    """The topn nearest other rows of every row of vectors [N, D] (device) by cosine: (ids, values) [N, topn] as device
    tensors, padded with (INT_MAX, -inf).  Each row's query is its own unit-normalised vector, and only its own row is
    excluded: two rows with identical vectors are each other's nearest."""
    if topn + 1 > MAX_CANDIDATES:
        raise ValueError("--topn may be at most %d" % (MAX_CANDIDATES - 1))
    nn.bind(vectors, math)
    n = int(vectors.shape[0])
    q = nn.queries(np.arange(n), np.ones(n, dtype=np.float32), np.arange(n + 1))
    return nn.search(q, topn, exclude_self=True)


def nearest_rows(nn: NearestNeighbours, vectors, topn: int, math: int):
    """nearest_rows_device with (ids, values) on the host."""
    idx, val = nearest_rows_device(nn, vectors, topn, math)
    return idx.cpu().numpy(), val.cpu().numpy()
