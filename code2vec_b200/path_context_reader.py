"""Reader / tensoriser with the reference's surface (reference path_context_reader.py),
TensorFlow-free: `.c2v` text lines -> int32 index arrays + float32 mask, batched on the host for
the engine's host-buffer entry points.

Semantics restated from the reference (file:line = path_context_reader.py):
  * a line has exactly MAX_CONTEXTS + 1 space-separated fields; field 0 is the target name,
    the rest are `source,path,target` triples; empty fields are padding          (:79-83,122-125)
  * empty target -> the target vocab's OOV word; empty context -> "PAD,PAD,PAD"    (:79-83)
  * a context is split on ',' without skipping empties; missing pieces become the token PAD
    word                                                                           (:189-196)
  * the three parts are looked up with OOV as the default index                    (:205-207)
  * mask = 1.0 iff any of the three indices differs from its vocab's PAD index     (:210-214)
  * train/evaluate drop rows with no valid context; train also drops rows whose target is
    OOV                                                                            (:147,153-177)
  * train: repeat(NUM_TRAIN_EPOCHS) -> shuffle(SHUFFLE_BUFFER_SIZE) -> parse -> filter ->
    batch (last batch may be short); predict: one unfiltered row, batch axis 1     (:119-151,96-107)
A "dataset" here is a Python iterable of batches in the model's input form (numpy arrays), which
replaces the tf.data iterator; end of data is the end of iteration instead of OutOfRangeError.

Two tensorisers implement the same semantics: the pure-Python one below (always used for predict,
which needs the per-context strings) and the native one (native/batcher.cpp: multi-threaded C++
parse + hash lookups straight into numpy / pinned buffers) used for train / evaluate files.
tests/test_reader_native.py checks they agree row for row.
"""
from __future__ import annotations

import abc
import os
from enum import Enum
from typing import Iterable, Iterator, List, NamedTuple, Optional

import numpy as np

import ctypes as C

from .config import Config
from .vocabularies import Code2VecVocabs

_native_lib = None


def load_native_tensoriser():
    """ctypes handle of libc2v_batcher.so (built on first use with g++), or None if it cannot be built."""
    global _native_lib
    if _native_lib is None:
        try:
            from .native import build_native
            lib = C.CDLL(build_native.build())
            P, I32, I64 = C.c_void_p, C.c_int32, C.c_int64
            lib.c2v_vocab_create.restype = P
            lib.c2v_vocab_create.argtypes = [P, P, P, I64, I32, I32]
            lib.c2v_vocab_destroy.restype = None
            lib.c2v_vocab_destroy.argtypes = [P]
            lib.c2v_vocab_lookup.restype = I32
            lib.c2v_vocab_lookup.argtypes = [P, C.c_char_p, I64]
            if hasattr(lib, "c2v_pool_take"):
                lib.c2v_pool_take.restype = I32
                lib.c2v_pool_take.argtypes = [P, P, P, P, P, I64, I32, P, I32, P, P, P, P, P, I32]
            lib.c2v_parse_chunk.restype = I64
            lib.c2v_parse_chunk.argtypes = [P, I64, I32, P, P, P, I32, I32, I64, P, P, P, P, P, P, P, P, C.POINTER(I32)]
            _native_lib = lib
        except Exception:
            _native_lib = False
    return _native_lib or None


_INT64_MIN = -(1 << 63)


class _Chunk:
    """A file buffer and the number of leading bytes that are complete lines (what the tensoriser is given)."""
    __slots__ = ("buf", "n")

    def __init__(self, buf: bytes, n: int):
        self.buf, self.n = buf, n


_SCAN_BYTES = 1 << 16          # the backward scan for a chunk's last newline reads this many bytes at a time
_PEEK_BYTES = 1 << 12          # the forward scan for a share's first line start


def _rfind(fd: int, lo: int, hi: int, pred) -> int:
    """The highest position p in [lo, hi) of file fd whose block satisfies pred(block) -> index within the block, or -1;
    blocks are read backwards from hi."""
    while hi > lo:
        a = max(lo, hi - _SCAN_BYTES)
        blk = os.pread(fd, hi - a, a)
        i = pred(blk)
        if i >= 0:
            return a + i
        hi = a
    return -1


def chunk_ranges(fd: int, chunk_bytes: int):
    """The byte ranges [a, b) of the chunks one pass of _native_chunks reads from file fd: a window of chunk_bytes from
    the end of the previous chunk is cut after its last newline; a window without one (a line longer than it) is retried
    twice as large, and the larger window stays; the window that reaches the end of the file is the last chunk whole,
    unless it holds no newline and nothing but '\\r' bytes, which yields nothing.  Each cut is found by reading the
    window backwards from its end, so a chunk's bytes are not read here."""
    end = os.fstat(fd).st_size
    start, size = 0, int(chunk_bytes)
    clean = 0                                  # [start, clean) is known to hold no newline
    while start < end:
        if end - start < size:                 # the window reaches the end of the file
            if _rfind(fd, start, end, lambda blk: len(blk.rstrip(b"\r")) - 1) >= 0:
                yield start, end
            return
        cut = _rfind(fd, max(start, clean), start + size, lambda blk: blk.rfind(b"\n"))
        if cut < 0:
            clean = start + size
            size *= 2
            continue
        yield start, cut + 1
        start = clean = cut + 1


def line_start_at_or_after(fd: int, t: int, a: int, b: int) -> int:
    """The first line start p >= t of the chunk [a, b) of file fd (p == a, or byte p - 1 is a newline); b if none."""
    if t <= a:
        return a
    p = t - 1
    while p < b:
        blk = os.pread(fd, min(_PEEK_BYTES, b - p), p)
        i = blk.find(b"\n")
        if i >= 0:
            return p + i + 1
        p += len(blk)
    return b


def share_range(fd: int, a: int, b: int, world: int, rank: int):
    """Rank `rank`'s share [s0, s1) of the chunk [a, b) of file fd among `world` ranks: from the first line start at or
    after a + rank (b - a) / world to the next rank's start (b for the last rank).  Shares are whole lines in rank order
    and cover the chunk; a line that spans a split point leaves the shares it swallows empty."""
    split = lambda r: line_start_at_or_after(fd, a + r * (b - a) // world, a, b)
    return split(rank), (b if rank == world - 1 else split(rank + 1))


def pread_into(fd: int, out, offset: int):
    """Fills the writable buffer `out` with the file's bytes from `offset` (os.preadv: no intermediate copy)."""
    mv = memoryview(out).cast("B")
    done = 0
    while done < len(mv):
        n = os.preadv(fd, [mv[done:]], offset + done)
        if n <= 0:
            raise EOFError("the data file ended %d bytes short of a chunk it was cut into" % (len(mv) - done))
        done += n


def _raise_parse_error(n: int, kind: int, max_contexts: int):
    """c2v_parse_chunk's negative return values as the reader's ValueErrors."""
    if n == _INT64_MIN:
        # more records than a chunk of that many bytes can hold well-formed lines: some line is far too short
        raise ValueError("Expect %d fields but have a different number in record (a line of the chunk is too short)"
                         % (max_contexts + 1))
    if kind == 2:
        raise ValueError("a context has more than 3 comma-separated parts (line %d of the chunk)" % (-n - 1))
    raise ValueError("Expect %d fields but have a different number in record (line %d of the chunk)" % (max_contexts + 1, -n - 1))


class _NativeVocab:
    def __init__(self, lib, vocab):
        self.lib = lib
        words = list(vocab.word_to_index.keys())
        enc = [w.encode("utf-8") for w in words]
        offsets = np.zeros(len(enc) + 1, dtype=np.int64)
        np.cumsum([len(b) for b in enc], out=offsets[1:])
        blob = b"".join(enc)
        idx = np.fromiter((vocab.word_to_index[w] for w in words), dtype=np.int32, count=len(words))
        pad_word = getattr(vocab.special_words, "PAD", vocab.special_words.OOV)
        self.h = lib.c2v_vocab_create(blob, offsets.ctypes.data, idx.ctypes.data, len(words),
                                      vocab.word_to_index[vocab.special_words.OOV], vocab.word_to_index[pad_word])

    def __del__(self):
        try:
            self.lib.c2v_vocab_destroy(self.h)
        except Exception:
            pass


class EstimatorAction(Enum):
    Train = "train"
    Evaluate = "evaluate"
    Predict = "predict"

    @property
    def is_train(self):
        return self is EstimatorAction.Train

    @property
    def is_evaluate(self):
        return self is EstimatorAction.Evaluate

    @property
    def is_predict(self):
        return self is EstimatorAction.Predict

    @property
    def is_evaluate_or_predict(self):
        return self.is_evaluate or self.is_predict


class ReaderInputTensors(NamedTuple):
    """Named access to the parts of one example or one batch (numpy arrays / lists of str)."""
    path_source_token_indices: np.ndarray
    path_indices: np.ndarray
    path_target_token_indices: np.ndarray
    context_valid_mask: np.ndarray
    target_index: Optional[np.ndarray] = None
    target_string: Optional[object] = None
    path_source_token_strings: Optional[object] = None
    path_strings: Optional[object] = None
    path_target_token_strings: Optional[object] = None


class ModelInputTensorsFormer(abc.ABC):
    """Implemented by the model: converts between ReaderInputTensors and the tuple it consumes."""

    @abc.abstractmethod
    def to_model_input_form(self, input_tensors: ReaderInputTensors):
        ...

    @abc.abstractmethod
    def from_model_input_form(self, input_row) -> ReaderInputTensors:
        ...


class PathContextReader:
    def __init__(self, vocabs: Code2VecVocabs, config: Config, model_input_tensors_former: ModelInputTensorsFormer,
                 estimator_action: EstimatorAction, repeat_endlessly: bool = False, shuffle_seed: Optional[int] = None,
                 keep_context_strings: Optional[bool] = None, use_native: Optional[bool] = None):
        self.vocabs = vocabs
        self.config = config
        self.model_input_tensors_former = model_input_tensors_former
        self.estimator_action = estimator_action
        self.repeat_endlessly = repeat_endlessly
        # bytes per chunk of the native path (chunk_ranges): where chunks end decides when the shuffle pool is drawn from
        self.chunk_bytes = 16 << 20
        tok, pth, tgt = vocabs.token_vocab, vocabs.path_vocab, vocabs.target_vocab
        self.CONTEXT_PADDING = ",".join([tok.special_words.PAD, pth.special_words.PAD, tok.special_words.PAD])
        self.csv_record_defaults = [[tgt.special_words.OOV]] + ([[self.CONTEXT_PADDING]] * config.MAX_CONTEXTS)
        self.create_needed_vocabs_lookup_tables(vocabs)
        self._tok_pad_word = tok.special_words.PAD
        self._pth_pad_word = pth.special_words.PAD
        self._tok_pad = tok.word_to_index[tok.special_words.PAD]
        self._pth_pad = pth.word_to_index[pth.special_words.PAD]
        self._tok_oov = tok.word_to_index[tok.special_words.OOV]
        self._pth_oov = pth.word_to_index[pth.special_words.OOV]
        self._tgt_oov_word = tgt.special_words.OOV
        self._tgt_oov = tgt.word_to_index[tgt.special_words.OOV]
        self._rng = np.random.default_rng(shuffle_seed)
        # evaluate() never reads the per-context strings; predict() needs them for the attention dict
        self.keep_context_strings = estimator_action.is_predict if keep_context_strings is None else keep_context_strings
        self._dataset = None
        self.use_native = use_native
        self._native = None

    @classmethod
    def create_needed_vocabs_lookup_tables(cls, vocabs: Code2VecVocabs):
        vocabs.token_vocab.get_word_to_index_lookup_table()
        vocabs.path_vocab.get_word_to_index_lookup_table()
        vocabs.target_vocab.get_word_to_index_lookup_table()

    # ---- one line -> one example -----------------------------------------------------------------
    def _split_row(self, row: str) -> List[str]:
        fields = row.rstrip("\r\n").split(" ")
        want = self.config.MAX_CONTEXTS + 1
        if len(fields) != want:
            raise ValueError("Expect %d fields but have %d in record" % (want, len(fields)))
        return fields

    def _map_raw_dataset_row_to_input_tensors(self, *row_parts) -> ReaderInputTensors:
        C = self.config.MAX_CONTEXTS
        tok_get = self.vocabs.token_vocab.word_to_index.get
        pth_get = self.vocabs.path_vocab.word_to_index.get
        target_str = row_parts[0] if row_parts[0] != "" else self._tgt_oov_word
        target_index = np.int32(self.vocabs.target_vocab.word_to_index.get(target_str, self._tgt_oov))
        src = np.full(C, self._tok_pad, dtype=np.int32)
        pth = np.full(C, self._pth_pad, dtype=np.int32)
        tgt = np.full(C, self._tok_pad, dtype=np.int32)
        keep = self.keep_context_strings
        if keep:
            s_str, p_str, t_str = [self._tok_pad_word] * C, [self._pth_pad_word] * C, [self._tok_pad_word] * C
        tok_oov, pth_oov, tok_pad_word = self._tok_oov, self._pth_oov, self._tok_pad_word
        for c in range(C):
            field = row_parts[c + 1]
            if field == "":
                continue                         # default "PAD,PAD,PAD": indices stay PAD
            pieces = field.split(",")
            n = len(pieces)
            if n > 3:
                raise ValueError("context %r has more than 3 comma-separated parts" % field)
            s = pieces[0]
            p = pieces[1] if n > 1 else tok_pad_word   # missing pieces are filled with the token PAD word (:193-196)
            t = pieces[2] if n > 2 else tok_pad_word
            src[c] = tok_get(s, tok_oov)
            pth[c] = pth_get(p, pth_oov)
            tgt[c] = tok_get(t, tok_oov)
            if keep:
                s_str[c], p_str[c], t_str[c] = s, p, t
        mask = ((src != self._tok_pad) | (tgt != self._tok_pad) | (pth != self._pth_pad)).astype(np.float32)
        return ReaderInputTensors(
            path_source_token_indices=src, path_indices=pth, path_target_token_indices=tgt, context_valid_mask=mask,
            target_index=target_index, target_string=target_str,
            path_source_token_strings=s_str if keep else None, path_strings=p_str if keep else None,
            path_target_token_strings=t_str if keep else None)

    def _filter_input_rows(self, row: ReaderInputTensors) -> bool:
        any_valid = (row.path_source_token_indices.max() != self._tok_pad
                     or row.path_target_token_indices.max() != self._tok_pad
                     or row.path_indices.max() != self._pth_pad)
        if self.estimator_action.is_evaluate:
            return bool(any_valid)
        return bool(any_valid and row.target_index > self._tgt_oov)

    @staticmethod
    def _stack(rows: List[ReaderInputTensors]) -> ReaderInputTensors:
        def col(name):
            vals = [getattr(r, name) for r in rows]
            if vals[0] is None:
                return None
            if isinstance(vals[0], np.ndarray) or np.isscalar(vals[0]) and not isinstance(vals[0], str):
                return np.stack(vals, axis=0) if isinstance(vals[0], np.ndarray) else np.asarray(vals, dtype=np.int32)
            return vals
        return ReaderInputTensors(**{name: col(name) for name in ReaderInputTensors._fields})

    def process_input_row(self, row_placeholder: str):
        """One line -> the model's input form with a leading batch axis of 1.  No row filter."""
        tensors = self._map_raw_dataset_row_to_input_tensors(*self._split_row(row_placeholder))
        return self.model_input_tensors_former.to_model_input_form(self._stack([tensors]))

    def process_and_iterate_input_from_data_lines(self, input_data_lines: Iterable) -> Iterable:
        for data_row in input_data_lines:
            yield self.process_input_row(data_row)

    # ---- the dataset pipeline ------------------------------------------------------------------------
    def get_dataset(self, input_data_rows: Optional[Iterable[str]] = None):
        if self._dataset is None:
            self._dataset = _BatchDataset(self, input_data_rows)
        return self._dataset

    def _raw_lines(self, input_data_rows) -> Iterator[str]:
        action = self.estimator_action

        def one_pass():
            if input_data_rows is not None:
                yield from input_data_rows
            else:
                assert not action.is_predict
                with open(self.config.data_path(is_evaluating=action.is_evaluate), "r",
                          buffering=max(1 << 16, min(self.config.CSV_BUFFER_SIZE or (1 << 20), 1 << 24))) as f:
                    yield from f

        if self.repeat_endlessly:
            while True:
                yield from one_pass()
        elif action.is_train and self.config.NUM_TRAIN_EPOCHS > 1:
            for _ in range(self.config.NUM_TRAIN_EPOCHS):
                yield from one_pass()
        else:
            yield from one_pass()

    def _shuffled(self, lines: Iterator[str]) -> Iterator[str]:
        """tf.data `shuffle(buffer)`: keep a buffer, emit a uniformly chosen element, refill."""
        size = max(int(self.config.SHUFFLE_BUFFER_SIZE), 1)
        buf: List[str] = []
        for line in lines:
            if len(buf) < size:
                buf.append(line)
                continue
            j = int(self._rng.integers(0, size))
            out, buf[j] = buf[j], line
            yield out
        self._rng.shuffle(buf)
        yield from buf

    # ---- native tensoriser path (train / evaluate over files) -----------------------------------------
    def _native_ready(self) -> bool:
        if self.use_native is False or self.estimator_action.is_predict or self.keep_context_strings:
            return False
        if self._native is None:
            lib = load_native_tensoriser()
            if lib is None:
                if self.use_native:
                    raise RuntimeError("native tensoriser requested but libc2v_batcher.so could not be built")
                self._native = False
            else:
                self._native = (lib, _NativeVocab(lib, self.vocabs.token_vocab), _NativeVocab(lib, self.vocabs.path_vocab),
                                _NativeVocab(lib, self.vocabs.target_vocab))
        return bool(self._native)

    def _native_parse(self, chunk):
        """bytes of complete lines -> (ReaderInputTensors of all rows, keep mask, target strings or None)."""
        lib, tok, pth, tgt = self._native
        Cn = self.config.MAX_CONTEXTS
        data, nbytes = (chunk.buf, chunk.n) if isinstance(chunk, _Chunk) else (chunk, len(chunk))
        cap = nbytes // (Cn + 1) + 1              # a line is at least MAX_CONTEXTS spaces + a newline long
        bufs = getattr(self, "_parse_bufs", None)
        if bufs is None or bufs[0].shape[0] < cap:   # scratch reused across chunks (no page faults per chunk)
            bufs = (np.empty((cap, Cn), dtype=np.int32), np.empty((cap, Cn), dtype=np.int32),
                    np.empty((cap, Cn), dtype=np.int32), np.empty((cap, Cn), dtype=np.float32),
                    np.empty(cap, dtype=np.int32), np.zeros(cap, dtype=np.uint8), np.empty(cap, dtype=np.int64),
                    np.empty(cap, dtype=np.int32))
            self._parse_bufs = bufs
        src, path, dst, mask, target, keep, toff, tlen = bufs
        cap = src.shape[0]
        err = C.c_int32(0)
        mode = 0 if self.estimator_action.is_train else 1
        threads = max(1, int(self.config.READER_NUM_PARALLEL_BATCHES or 1))
        n = lib.c2v_parse_chunk(data, nbytes, Cn, tok.h, pth.h, tgt.h, mode, threads, cap, src.ctypes.data,
                                path.ctypes.data, dst.ctypes.data, mask.ctypes.data, target.ctypes.data, keep.ctypes.data,
                                toff.ctypes.data, tlen.ctypes.data, C.byref(err))
        if n < 0:
            _raise_parse_error(n, err.value, Cn)
        sel = keep[:n].astype(bool)
        strings = None
        if self.estimator_action.is_evaluate:
            oov = self._tgt_oov_word
            strings = [data[o:o + l].decode("utf-8") if l else oov for o, l, k in zip(toff[:n], tlen[:n], sel) if k]
        return (src[:n][sel], path[:n][sel], dst[:n][sel], mask[:n][sel], target[:n][sel]), strings

    def _native_parse_into(self, chunk, pool: "_RowPool"):
        """Train path: rows are parsed straight into the tail of the shuffle pool (no scratch copy, no
        selection copy); rows the filter drops are then overwritten by kept rows from the end."""
        lib, tok, pth, tgt = self._native
        Cn = self.config.MAX_CONTEXTS
        data, nbytes = (chunk.buf, chunk.n) if isinstance(chunk, _Chunk) else (chunk, len(chunk))
        cap = nbytes // (Cn + 1) + 1                 # a line is at least MAX_CONTEXTS spaces + a newline long; the
        #                                              reserve is address space only -- pages are touched as rows land
        pool.reserve(cap, Cn)
        small = getattr(self, "_parse_small", None)
        if small is None or small[0].shape[0] < cap:
            small = (np.zeros(cap, dtype=np.uint8), np.empty(cap, dtype=np.int64), np.empty(cap, dtype=np.int32))
            self._parse_small = small
        keep, toff, tlen = small
        src, path, dst, mask, target = pool.tail_pointers()
        err = C.c_int32(0)
        threads = max(1, int(self.config.READER_NUM_PARALLEL_BATCHES or 1))
        n = lib.c2v_parse_chunk(data, nbytes, Cn, tok.h, pth.h, tgt.h, 0, threads, cap, src, path, dst, mask, target,
                                keep.ctypes.data, toff.ctypes.data, tlen.ctypes.data, C.byref(err))
        if n < 0:
            _raise_parse_error(n, err.value, Cn)
        pool.commit(n, keep[:n])

    def _native_chunk_ranges(self):
        """(fd, a, b) for every chunk [a, b) of the data file (chunk_ranges), one pass per epoch like _raw_lines; fd is
        open until the next pass begins."""
        action = self.estimator_action
        path = self.config.data_path(is_evaluating=action.is_evaluate)
        passes = 1
        if action.is_train and not self.repeat_endlessly and self.config.NUM_TRAIN_EPOCHS > 1:
            passes = self.config.NUM_TRAIN_EPOCHS
        p = 0
        while self.repeat_endlessly or p < passes:
            p += 1
            with open(path, "rb") as f:
                fd = f.fileno()
                for a, b in chunk_ranges(fd, self.chunk_bytes):
                    yield fd, a, b

    def _native_chunks(self):
        """Complete-line byte chunks of the data file, one pass per epoch like _raw_lines."""
        for fd, a, b in self._native_chunk_ranges():
            buf = os.pread(fd, b - a, a)
            while len(buf) < b - a:                  # a short read: the rest follows
                more = os.pread(fd, b - a - len(buf), a + len(buf))
                if not more:
                    raise EOFError("the data file ended %d bytes short of a chunk it was cut into" % (b - a - len(buf)))
                buf += more
            yield _Chunk(buf, b - a)

    def _native_chunks_ahead(self, depth: int = 2):
        """_native_chunks read `depth` chunks ahead by a helper thread (file reads and the slicing of complete lines release
        the GIL), so the disk/page-cache read of chunk k+1 overlaps the tensorisation of chunk k."""
        import queue
        import threading
        q: "queue.Queue" = queue.Queue(maxsize=depth)
        done, stop = object(), threading.Event()

        def run():
            try:
                for chunk in self._native_chunks():
                    while not stop.is_set():
                        try:
                            q.put(chunk, timeout=0.1)
                            break
                        except queue.Full:
                            continue
                    if stop.is_set():
                        return
                q.put(done)
            except BaseException as exc:
                q.put(exc)

        threading.Thread(target=run, daemon=True).start()
        try:
            while True:
                item = q.get()
                if item is done:
                    return
                if isinstance(item, BaseException):
                    raise item
                yield item
        finally:
            stop.set()

    def _iterate_batches_native(self):
        action = self.estimator_action
        B = self.config.batch_size(is_evaluating=action.is_evaluate)
        former = self.model_input_tensors_former
        names = ("path_source_token_indices", "path_indices", "path_target_token_indices", "context_valid_mask", "target_index")

        def emit(arrs, strings):
            return former.to_model_input_form(ReaderInputTensors(target_string=strings, **dict(zip(names, arrs))))

        if action.is_evaluate:
            pend, pend_s = None, []
            for chunk in self._native_chunks():
                arrs, strings = self._native_parse(chunk)
                pend = arrs if pend is None else tuple(np.concatenate([a, b]) for a, b in zip(pend, arrs))
                pend_s += strings
                while pend[0].shape[0] >= B:
                    yield emit(tuple(a[:B] for a in pend), pend_s[:B])
                    pend, pend_s = tuple(a[B:] for a in pend), pend_s[B:]
            if pend is not None and pend[0].shape[0]:
                yield emit(pend, pend_s)
            return
        # train: a pool of at least SHUFFLE_BUFFER_SIZE rows; every batch is a uniform draw without
        # replacement from the pool (tf.data's shuffle(buffer) draws the same way, one row at a time)
        S = max(int(self.config.SHUFFLE_BUFFER_SIZE), 1)
        # one thread: the draw is ~8 MB of random row copies per batch and thread start-up cost more than it saved when measured
        pool = _RowPool(native=self._native[0], threads=1)
        ring = getattr(self, "batch_ring", None)          # PinnedBatchRing: batches are drawn straight into pinned slots

        def draw(b):
            if ring is None:
                return pool.take(b, self._rng)
            return pool.take(b, self._rng, out=ring.acquire().arrays())
        for chunk in self._native_chunks_ahead():
            self._native_parse_into(chunk, pool)
            while pool.n >= S + B:
                yield emit(draw(B), None)
        while pool.n > 0:
            yield emit(draw(min(B, pool.n)), None)

    def _iterate_batches(self, input_data_rows):
        action = self.estimator_action
        if input_data_rows is None and self._native_ready():
            yield from self._iterate_batches_native()
            return
        lines = self._raw_lines(input_data_rows)
        if action.is_train:
            lines = self._shuffled(lines)
        batch_size = 1 if action.is_predict else self.config.batch_size(is_evaluating=action.is_evaluate)
        rows: List[ReaderInputTensors] = []
        for line in lines:
            if line in ("", "\n"):
                continue
            row = self._map_raw_dataset_row_to_input_tensors(*self._split_row(line))
            if not action.is_predict and not self._filter_input_rows(row):
                continue
            rows.append(row)
            if len(rows) == batch_size:
                yield self.model_input_tensors_former.to_model_input_form(self._stack(rows))
                rows = []
        if rows:
            yield self.model_input_tensors_former.to_model_input_form(self._stack(rows))


class _RowPool:
    """Shuffle pool over parallel row arrays: O(rows appended) to add, O(batch) to draw -- drawn rows are
    replaced by rows from the tail, nothing else moves."""

    def __init__(self, native=None, threads: int = 1):
        self.arrays = None
        self.n = 0
        self.native = native if (native is not None and hasattr(native, "c2v_pool_take")) else None     # libc2v_batcher.so
        self.threads = max(1, int(threads))

    def append(self, arrs):
        k = arrs[0].shape[0]
        if k == 0:
            return
        if self.arrays is None:
            cap = max(2 * k, 1024)
            self.arrays = [np.empty((cap,) + a.shape[1:], dtype=a.dtype) for a in arrs]
        if self.n + k > self.arrays[0].shape[0]:
            cap = max(2 * self.arrays[0].shape[0], self.n + k)
            grown = [np.empty((cap,) + a.shape[1:], dtype=a.dtype) for a in self.arrays]
            for g, a in zip(grown, self.arrays):
                g[:self.n] = a[:self.n]
            self.arrays = grown
        for dst, a in zip(self.arrays, arrs):
            dst[self.n:self.n + k] = a
        self.n += k

    def reserve(self, k: int, contexts: int):
        """Room for k more rows behind the current end (arrays are created on first use: three int32 index
        matrices, the float32 mask, the int32 targets -- the reader's column order)."""
        if self.arrays is None:
            cap = max(2 * k, 1024)
            self.arrays = [np.empty((cap, contexts), dtype=np.int32), np.empty((cap, contexts), dtype=np.int32),
                           np.empty((cap, contexts), dtype=np.int32), np.empty((cap, contexts), dtype=np.float32),
                           np.empty((cap,), dtype=np.int32)]
        if self.n + k > self.arrays[0].shape[0]:
            cap = max(2 * self.arrays[0].shape[0], self.n + k)
            grown = [np.empty((cap,) + a.shape[1:], dtype=a.dtype) for a in self.arrays]
            for g, a in zip(grown, self.arrays):
                g[:self.n] = a[:self.n]
            self.arrays = grown

    def tail_pointers(self):
        """Addresses of row `n` in every array: where a parser may write reserved rows."""
        return tuple(a.ctypes.data + self.n * a.strides[0] for a in self.arrays)

    def commit(self, k: int, keep):
        """k rows were written behind the end; keep[i] == 0 marks rows to drop.  Dropped rows inside the new
        extent are overwritten by kept rows from beyond it -- O(dropped) row moves."""
        keep = np.asarray(keep[:k], dtype=bool)
        kept = int(keep.sum())
        if kept < k:
            holes = self.n + np.flatnonzero(~keep[:kept])
            movers = self.n + kept + np.flatnonzero(keep[kept:])
            if holes.size:
                for a in self.arrays:
                    a[holes] = a[movers]
        self.n += kept

    def take(self, b: int, rng, out=None) -> tuple:
        """b rows drawn uniformly without replacement.  out: five arrays with at least b rows (e.g. a page-locked batch
        slot) the rows are gathered into; the views of their first b rows are returned."""
        n = self.n
        pick = rng.choice(n, size=b, replace=False) if b < n else rng.permutation(n)
        if self.native is not None and self._native_layout(out, b):
            # one native call, row copies spread over the reader's threads: the same gather and the same hole filling as below
            if out is None:
                out = tuple(np.empty((b,) + a.shape[1:], dtype=a.dtype) for a in self.arrays)
            pick = np.ascontiguousarray(pick, dtype=np.int64)
            rc = self.native.c2v_pool_take(*(a.ctypes.data for a in self.arrays), n, self.arrays[0].shape[1], pick.ctypes.data, b,
                                           *(o.ctypes.data for o in out), self.threads)
            if rc != 0:
                raise RuntimeError("c2v_pool_take rejected the draw (%d rows of %d)" % (b, n))
            self.n = n - b
            return tuple(o[:b] for o in out)
        if out is None:
            out = tuple(a[pick] for a in self.arrays)
        else:
            for a, o in zip(self.arrays, out):
                np.take(a, pick, axis=0, out=o[:b], mode="clip")     # indices are in range; "raise" would buffer the output
            out = tuple(o[:b] for o in out)
        # fill the holes left below the new end with the surviving rows of the tail
        new_n = n - b
        chosen = np.zeros(n, dtype=bool)
        chosen[pick] = True
        holes = np.flatnonzero(chosen[:new_n])
        movers = new_n + np.flatnonzero(~chosen[new_n:])
        if holes.size:
            for a in self.arrays:
                a[holes] = a[movers]
        self.n = new_n
        return out


    def _native_layout(self, out, b: int) -> bool:
        """The native draw wants the reader's own column layout: three int32 [*, C] matrices, a float32 [*, C] mask, int32 targets,
        all C-contiguous, and out buffers (if given) of the same kind with at least b rows."""
        A = self.arrays
        if A is None or len(A) != 5:
            return False
        C = A[0].shape[1] if A[0].ndim == 2 else -1
        kinds = (np.int32, np.int32, np.int32, np.float32, np.int32)
        for i, (a, k) in enumerate(zip(A, kinds)):
            if a.dtype != k or not a.flags.c_contiguous or (a.ndim != (2 if i < 4 else 1)) or (i < 4 and a.shape[1] != C):
                return False
        if out is not None:
            if len(out) != 5:
                return False
            for i, (o, k) in enumerate(zip(out, kinds)):
                if (not isinstance(o, np.ndarray) or o.dtype != k or not o.flags.c_contiguous or o.shape[0] < b or
                        o.ndim != (2 if i < 4 else 1) or (i < 4 and o.shape[1] != C)):
                    return False
        return True


class _BatchDataset:
    """Re-iterable view: every `iter()` restarts the pipeline (the reference re-runs the iterator's
    initializer op before each evaluation, tensorflow_model.py:147)."""

    def __init__(self, reader: PathContextReader, input_data_rows):
        self.reader = reader
        self.input_data_rows = input_data_rows

    def __iter__(self):
        return self.reader._iterate_batches(self.input_data_rows)
