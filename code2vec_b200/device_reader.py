"""Training batches read on the GPU (DESIGN.md §6d): `.c2v` text chunks are uploaded as bytes, parsed, looked up in the
vocabularies and drawn from a shuffle pool in device memory by the reader kernels of libc2v_b200.so (include/c2v_b200.h,
"Device reader").  Every batch equals, row for row and bit for bit, the one PathContextReader._iterate_batches_native
yields in train mode for the same config and shuffle seed:
  * the file is read by the host reader's own chunker (_native_chunks_ahead: the long-line retry and a last line without
    a newline come with it);
  * the vocabularies are the native tensoriser's hash tables, copied to the device as they are (c2v_vocab_export);
  * the host draws every batch's row indices with the reader's np.random.Generator exactly as _RowPool.take does, and the
    pool on the device is committed and drawn from in the host pool's order, so the same indices pick the same rows.
The host's work per chunk is a file read, one copy into a page-locked buffer and its upload; per batch, the draw of the
indices (8 bytes a row).  Code2VecModel.train() uses it when C2V_DEVICE_READER=1.

Sharded (C2V_SHARDED_READER=1 on W > 1 ranks, a ShareTransport given): the ranks cut every chunk into W shares of whole
lines (path_context_reader.share_range); each rank reads, uploads and parses only its own share into a stage of its
device memory (c2v_reader_parse_share), the ranks gather their share statuses once per chunk, and every rank assembles
all W stages, its peers' read through CUDA IPC, into its pool (c2v_reader_commit_shares).  Chunk bounds, pool, kept
counts and draws stay exactly those of the unsharded reader, so the batches do too.

Evaluate mode (a PathContextReader with EstimatorAction.Evaluate; C2V_DEVICE_EVAL=1, DESIGN.md §6e): the test file is
parsed in device memory with the evaluate filter, the kept rows queue in file order with their names, and every batch is
the queue's next TEST_BATCH_SIZE rows -- the batches of _iterate_batches_native in evaluate mode, row for row, across
chunk boundaries.  score() runs the metric kernel on the engine's top-k ids of a batch and brings back only the per-row
results, the names and the integer accumulators."""
from __future__ import annotations

import ctypes as C
import datetime
import queue
import threading
from typing import Optional

import numpy as np

from .engine import EngineError, c2v_reader_share_status, c2v_reader_vocab, load_library
from .multi_rank import batch_split
from .path_context_reader import _INT64_MIN, PathContextReader, _raise_parse_error, pread_into, share_range

# how long a rank waits in a chunk's exchange for its peers (they may be evaluating, or saving a checkpoint)
EXCHANGE_TIMEOUT = datetime.timedelta(minutes=30)


def device_reader_flag(environ) -> bool:
    """C2V_DEVICE_READER=1: Code2VecModel.train() reads its batches on the GPU; 0 (the default): on the host."""
    flag = environ.get("C2V_DEVICE_READER", "0") or "0"
    if flag not in ("0", "1"):
        raise ValueError("C2V_DEVICE_READER must be 0 or 1, got %r" % flag)
    return flag == "1"


def device_eval_flag(environ) -> bool:
    """C2V_DEVICE_EVAL=1: Code2VecModel.evaluate() reads, predicts and scores on the GPU; 0 (the default): on the host."""
    flag = environ.get("C2V_DEVICE_EVAL", "0") or "0"
    if flag not in ("0", "1"):
        raise ValueError("C2V_DEVICE_EVAL must be 0 or 1, got %r" % flag)
    return flag == "1"


def evaluation_route_line(device_eval: bool) -> str:
    """The start-up log line of the evaluation route: evaluate(), --score_names and --nearest on the GPU or the host."""
    if device_eval:
        route = ("evaluate() read, predicted and scored on the GPU; --score_names and --nearest read, scored or searched "
                 "and written on the GPU")
    else:
        route = "evaluate(), --score_names and --nearest read and scored on the host"
    return "b200 backend evaluation: %s (C2V_DEVICE_EVAL=%d)" % (route, int(device_eval))


def sharded_reader_flag(environ) -> bool:
    """C2V_SHARDED_READER=1 (with C2V_DEVICE_READER=1): on several GPUs each rank reads and parses 1/W of every chunk and
    takes the other rows from its peers; 0 (the default): every rank reads the whole file."""
    flag = environ.get("C2V_SHARDED_READER", "0") or "0"
    if flag not in ("0", "1"):
        raise ValueError("C2V_SHARDED_READER must be 0 or 1, got %r" % flag)
    return flag == "1"


def chunk_error(statuses, chunk_bytes: int, max_contexts: int):
    """The error of a chunk parsed as shares, from the shares' statuses in rank order (objects with records, newlines,
    bad_line, bad_kind, overflow): None for a clean chunk, (None, 3) when the chunk has more records than
    chunk_bytes / (max_contexts + 1) + 1, else (line, kind) of its lowest malformed line -- what a whole-chunk parse
    reports."""
    cap = chunk_bytes // (max_contexts + 1) + 1
    if sum(s.records for s in statuses) > cap:
        return None, 3
    base = 0
    for s in statuses:
        if s.bad_kind:
            return base + s.bad_line, s.bad_kind
        if s.overflow:
            raise RuntimeError("a share overflowed its stage but reported no malformed line")
        base += s.newlines
    return None


def raise_chunk_error(err, max_contexts: int):
    """chunk_error's verdict as the ValueError the host reader raises for the same chunk."""
    line, kind = err
    if kind == 3:
        _raise_parse_error(_INT64_MIN, 0, max_contexts)
    _raise_parse_error(-(line + 1), kind, max_contexts)


class ShareTransport:
    """How the ranks of a sharded device reader meet: `gather` is an all-gather of one small object per rank on a gloo
    group of the reader's own (the reader thread never issues a collective on the training group, whose NCCL
    collectives the training thread issues at the same time), and stages are CUDA-IPC allocations that peers open by
    handle.  Tests replace it (make_share_transport) to run ranks as threads of one process."""

    def __init__(self, lib, device: int, group, world: int, rank: int):
        self.lib, self.device, self.group, self.world, self.rank = lib, int(device), group, int(world), int(rank)

    def _check(self, rc):
        if rc != 0:
            raise EngineError(rc, self.lib.c2v_last_error(None).decode())

    def alloc(self, nbytes: int):
        """(device pointer, handle bytes) of a new peer-visible allocation on this rank's device."""
        ptr, hbuf = C.c_void_p(), C.create_string_buffer(64)
        self._check(self.lib.c2v_ipc_alloc(self.device, nbytes, C.byref(ptr), hbuf))
        return ptr.value, hbuf.raw

    def free(self, ptr: int):
        self._check(self.lib.c2v_ipc_free(self.device, ptr))

    def open(self, handle: bytes) -> int:
        ptr = C.c_void_p()
        self._check(self.lib.c2v_ipc_open(self.device, handle, C.byref(ptr)))
        return ptr.value

    def close(self, ptr: int):
        self._check(self.lib.c2v_ipc_close(self.device, ptr))

    def gather(self, obj) -> list:
        import torch.distributed as dist
        out = [None] * self.world
        dist.all_gather_object(out, obj, group=self.group)
        return out

    def destroy(self):
        import torch.distributed as dist
        if self.group is not None:
            dist.destroy_process_group(self.group)
            self.group = None


def make_share_transport(device: int) -> ShareTransport:
    """The transport of a sharded reader on this rank of the default process group (every rank calls it, in the same
    order as its other new_group calls)."""
    import torch.distributed as dist
    group = dist.new_group(backend="gloo", timeout=EXCHANGE_TIMEOUT)
    return ShareTransport(load_library(), device, group, dist.get_world_size(), dist.get_rank())


def export_vocab(lib, handle):
    """(slots [mask + 1, 24] uint8, word bytes uint8, mask, oov, pad) of a native vocabulary (c2v_vocab_export), as numpy
    views of the table's own memory (valid while the vocabulary lives)."""
    if not hasattr(lib, "c2v_vocab_export"):
        raise RuntimeError("libc2v_batcher.so has no c2v_vocab_export: rebuild it (code2vec_b200/native/build_native.py)")
    fn = lib.c2v_vocab_export
    fn.restype = None
    fn.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.POINTER(C.c_void_p),
                   C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    slots, mask, words, n_bytes, oov, pad = C.c_void_p(), C.c_uint64(), C.c_void_p(), C.c_int64(), C.c_int32(), C.c_int32()
    fn(handle, C.byref(slots), C.byref(mask), C.byref(words), C.byref(n_bytes), C.byref(oov), C.byref(pad))
    n_slots = int(mask.value) + 1
    slot_arr = np.ctypeslib.as_array((C.c_uint8 * (24 * n_slots)).from_address(slots.value)).reshape(n_slots, 24)
    byte_arr = (np.ctypeslib.as_array((C.c_uint8 * n_bytes.value).from_address(words.value)) if n_bytes.value
                else np.zeros(0, dtype=np.uint8))
    return slot_arr, byte_arr, int(mask.value), int(oov.value), int(pad.value)


class DeviceVocabs:
    """The native tensoriser's three vocabularies (c2v_vocab_export) copied to one device, with the c2v_reader_vocab
    structs that point at them.  One model uploads them once and shares them between its training and evaluation readers
    (about 165 MB at java14m size); `reader` is any PathContextReader of the model with the native tensoriser ready."""

    def __init__(self, reader: PathContextReader, device):
        import torch
        lib_b, tok, pth, tgt = reader._native
        self.dev = torch.device(device)
        self.tensors, self.structs = [], []
        with torch.cuda.device(self.dev):
            for v in (tok, pth, tgt):
                slot_arr, byte_arr, mask, oov, pad = export_vocab(lib_b, v.h)
                d_slots = torch.from_numpy(slot_arr).to(self.dev)
                d_bytes = torch.from_numpy(byte_arr if byte_arr.size else np.zeros(1, dtype=np.uint8)).to(self.dev)
                self.tensors += [d_slots, d_bytes]
                self.structs.append(c2v_reader_vocab(d_slots.data_ptr(), d_bytes.data_ptr(), mask, oov, pad))
            torch.cuda.synchronize(self.dev)

    def nbytes(self) -> int:
        return int(sum(t.numel() * t.element_size() for t in self.tensors))


def eval_tables(target_vocab):
    """The per-target-word tables of the metric kernel (c2v_reader_eval_tables), computed with the host metrics' own
    functions: (words, word_off, norm, norm_off, legal) -- every word's UTF-8 bytes, its common.normalize_word bytes and
    common.legal_method_names_checker, as numpy arrays."""
    from .common import common
    special = target_vocab.special_words
    words = [target_vocab.index_to_word[i] for i in range(target_vocab.size)]
    enc = [w.encode("utf-8") for w in words]
    norm = [common.normalize_word(w).encode("utf-8") for w in words]
    legal = np.fromiter((bool(common.legal_method_names_checker(special, w)) for w in words), dtype=np.uint8,
                        count=len(words))

    def packed(items):
        off = np.zeros(len(items) + 1, dtype=np.int64)
        np.cumsum([len(b) for b in items], out=off[1:])
        return np.frombuffer(b"".join(items) or b"\0", dtype=np.uint8), off
    w, w_off = packed(enc)
    n, n_off = packed(norm)
    return w, w_off, n, n_off, legal


class EvalScores:
    """What the metric kernel returns to the host for one batch of n rows: rank, first, flags [n] int32 (as
    c2v_reader_eval_score defines them), acc [k + 4] int64 (rank histogram, rows, tp, fp, fn of the rows scored on the
    device), and the rows' names (bytes).  ids [n, k] int32 only when a row is flagged: the host scores those rows."""
    __slots__ = ("rank", "first", "flags", "acc", "names", "ids")

    def __init__(self, rank, first, flags, acc, names, ids):
        self.rank, self.first, self.flags, self.acc, self.names, self.ids = rank, first, flags, acc, names, ids


class DeviceBatch:
    """One batch in a device slot: `tensors` = (src, path, tgt [rows, C] int32, mask [rows, C] float32, target [rows]
    int32) holding rows [lo, hi) of a global batch of `rows` rows (all of it on one GPU); `dropped` rows of a short batch
    are left out on several ranks (multi_rank.batch_split).  wait() makes the current stream wait for the draw; release()
    hands the slot back once the work queued so far on the current stream (the step that read it) is done.  An
    evaluation batch also has its rows' names on the device (score() reads them)."""
    __slots__ = ("tensors", "rows", "lo", "hi", "dropped", "_slot", "_reader")

    def __init__(self, slot, rows, lo, hi, dropped, reader):
        self._slot, self._reader = slot, reader
        self.rows, self.lo, self.hi, self.dropped = rows, lo, hi, dropped
        self.tensors = tuple(t[:hi - lo] for t in slot["tensors"])

    def wait(self):
        torch = self._reader.torch
        torch.cuda.current_stream(self._reader.dev).wait_event(self._slot["ready"])

    def release(self):
        torch = self._reader.torch
        self._slot["done"].record(torch.cuda.current_stream(self._reader.dev))
        self._slot["free"].set()


class DeviceBatchReader:
    """Iterable of DeviceBatch for one training pass of `reader` (a train-mode PathContextReader; its shuffle seed and
    config decide every batch).  world / rank: this rank's slice of each global batch.  A reader thread uploads and parses
    the chunks and queues the draws into `slots` device slots, each reused only after the step that last read it; the
    iterating (training) thread never waits for the GPU.  Needs libc2v_batcher.so (RuntimeError otherwise, as
    use_native=True does).  With an evaluate-mode `reader` the slots are filled by sequential takes from the evaluation
    queue (no draws, no RNG), and the reader may be iterated again once a pass has ended."""

    def __init__(self, reader: PathContextReader, device, world: int = 1, rank: int = 0, slots: int = 4,
                 transport: Optional[ShareTransport] = None, vocabs: Optional[DeviceVocabs] = None, tables=None,
                 check_utf8: bool = False):
        """transport: read the chunks sharded across the `world` ranks, meeting through it (ignored on one rank).
        vocabs: the model's DeviceVocabs (uploaded here when None).  tables: eval_tables(target vocabulary), needed by
        an evaluation reader (an evaluate-mode `reader`); every rank of an evaluation reads the whole file.  check_utf8
        (evaluation): each chunk's names are checked as the host reader decodes them, so a name that is not valid UTF-8
        raises the host reader's UnicodeDecodeError at the same chunk."""
        import torch
        action = reader.estimator_action
        if not (action.is_train or action.is_evaluate):
            raise ValueError("the device reader reads training and evaluation files only")
        self.evaluate = action.is_evaluate
        self.check_utf8 = bool(check_utf8)
        if self.evaluate and tables is None:
            raise ValueError("an evaluation reader needs the target-word tables (device_reader.eval_tables)")
        if slots < 3:
            raise ValueError("the device reader needs at least 3 batch slots")
        reader.use_native = True
        reader._native_ready()                 # RuntimeError when libc2v_batcher.so cannot be built
        self.torch, self.reader = torch, reader
        self.dev = torch.device(device)
        self.lib = load_library()
        self.world, self.rank = int(world), int(rank)
        cfg = reader.config
        self.C = int(cfg.MAX_CONTEXTS)
        self.B = int(cfg.batch_size(is_evaluating=self.evaluate))
        self.S = max(int(cfg.SHUFFLE_BUFFER_SIZE), 1)
        self.h2d_bytes = 0
        self.vocabs = vocabs if vocabs is not None else DeviceVocabs(reader, self.dev)
        self._own_vocabs = vocabs is None
        structs = self.vocabs.structs
        self._structs = structs
        with torch.cuda.device(self.dev):
            h = C.c_void_p()
            rc = self.lib.c2v_reader_create(self.C, C.byref(structs[0]), C.byref(structs[1]), C.byref(structs[2]),
                                            self.dev.index or 0, C.byref(h))
            if rc != 0:
                raise EngineError(rc, self.lib.c2v_last_error(None).decode())
            self.h = h
            self.stream = torch.cuda.Stream(device=self.dev)
            self.copy_stream = torch.cuda.Stream(device=self.dev)
            self._name_bytes = 0                   # evaluate: the bound on a take's name bytes (c2v_reader_eval_append)
            self.table_bytes = 0
            if self.evaluate:
                w, w_off, n, n_off, legal = tables
                rc = self.lib.c2v_reader_eval_tables(self.h, int(legal.size), w.ctypes.data, w_off.ctypes.data,
                                                     n.ctypes.data, n_off.ctypes.data, legal.ctypes.data,
                                                     self.stream.cuda_stream)
                if rc != 0:
                    raise EngineError(rc, self.lib.c2v_last_error(None).decode())
            local = self.B if self.evaluate else self.B // self.world
            self.slots = []
            for _ in range(slots):
                s = {"tensors": (torch.empty((local, self.C), dtype=torch.int32, device=self.dev),
                                 torch.empty((local, self.C), dtype=torch.int32, device=self.dev),
                                 torch.empty((local, self.C), dtype=torch.int32, device=self.dev),
                                 torch.empty((local, self.C), dtype=torch.float32, device=self.dev),
                                 torch.empty((local,), dtype=torch.int32, device=self.dev)),
                     "pick": torch.empty(self.B, dtype=torch.int64).pin_memory(),
                     "ready": torch.cuda.Event(), "done": torch.cuda.Event(), "free": threading.Event()}
                if self.evaluate:
                    s["name_off"] = torch.empty(self.B + 1, dtype=torch.int64, device=self.dev)
                    s["names"] = torch.empty(1 << 16, dtype=torch.uint8, device=self.dev)
                s["free"].set()
                self.slots.append(s)
        # chunk text: two page-locked buffers and two device buffers, so the upload of chunk k+1 overlaps the draws of k
        self._text = [None, None]
        self._thread: Optional[threading.Thread] = None
        self._stop = threading.Event()
        # sharded: this rank's two stages (chunk k uses stage k % 2), the peers' stages opened by handle, and replaced
        # stages waiting until no peer has them open
        self.transport = transport if self.world > 1 else None
        self._stages = [None, None]
        self._peers = {}                       # (rank, stage) -> opened pointer
        self._retired = []                     # (pointer, exchanges after which it is freed)
        self._exchanges = 0
        self._peers_know = False               # the peers know this rank is done with the pass's exchanges
        self.peer_bytes = 0                    # bytes of rows this rank's assemblies read from its peers' stages
        self._row_bytes = (4 * self.C + 1) * 4 + 1

    # ---- reader thread ---------------------------------------------------------------------------------------------
    def _text_buffers(self, i: int, n: int):
        torch = self.torch
        buf = self._text[i]
        if buf is None or buf["host"].numel() < n:
            if buf is not None:
                buf["uploaded"].synchronize()
            cap = max(n, 16 << 20)
            buf = {"host": torch.empty(cap, dtype=torch.uint8).pin_memory(),
                   "dev": torch.empty(cap, dtype=torch.uint8, device=self.dev), "uploaded": torch.cuda.Event()}
            buf["np"] = buf["host"].numpy()
            buf["uploaded"].record(self.copy_stream)
            self._text[i] = buf
        return buf

    def _parse(self, chunk, i: int) -> int:
        torch = self.torch
        n = int(chunk.n)
        buf = self._text_buffers(i, n)
        buf["uploaded"].synchronize()                       # the previous upload out of this host buffer has left
        buf["np"][:n] = np.frombuffer(chunk.buf, dtype=np.uint8, count=n)
        with torch.cuda.stream(self.copy_stream):
            buf["dev"][:n].copy_(buf["host"][:n], non_blocking=True)
            buf["uploaded"].record(self.copy_stream)
        self.stream.wait_event(buf["uploaded"])
        self.h2d_bytes += n
        kept, bad_line, bad_kind = C.c_int64(), C.c_int64(), C.c_int32()
        rc = self.lib.c2v_reader_parse_chunk(self.h, buf["dev"].data_ptr(), n, C.byref(kept), C.byref(bad_line),
                                             C.byref(bad_kind), self.stream.cuda_stream)
        if rc != 0:
            if bad_kind.value == 3:
                _raise_parse_error(_INT64_MIN, 0, self.C)
            if bad_kind.value in (1, 2):
                _raise_parse_error(-(bad_line.value + 1), bad_kind.value, self.C)
            raise EngineError(rc, self.lib.c2v_last_error(None).decode())
        return int(kept.value)

    # ---- evaluate mode -------------------------------------------------------------------------------------------------
    def _append(self, chunk, i: int) -> int:
        """Chunk `chunk` uploaded from host buffer i and appended to the evaluation queue; returns the rows kept."""
        torch = self.torch
        n = int(chunk.n)
        buf = self._text_buffers(i, n)
        buf["uploaded"].synchronize()
        buf["np"][:n] = np.frombuffer(chunk.buf, dtype=np.uint8, count=n)
        with torch.cuda.stream(self.copy_stream):
            buf["dev"][:n].copy_(buf["host"][:n], non_blocking=True)
            buf["uploaded"].record(self.copy_stream)
        self.stream.wait_event(buf["uploaded"])
        self.h2d_bytes += n
        kept, name_bytes, bad_line, bad_kind = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int32()
        rc = self.lib.c2v_reader_eval_append(self.h, buf["dev"].data_ptr(), n, C.byref(kept), C.byref(name_bytes),
                                             C.byref(bad_line), C.byref(bad_kind), self.stream.cuda_stream)
        if rc != 0:
            if bad_kind.value == 3:
                _raise_parse_error(_INT64_MIN, 0, self.C)
            if bad_kind.value in (1, 2):
                _raise_parse_error(-(bad_line.value + 1), bad_kind.value, self.C)
            raise EngineError(rc, self.lib.c2v_last_error(None).decode())
        self._name_bytes = int(name_bytes.value)
        if self.check_utf8 and kept.value:
            self._check_utf8(int(kept.value))
        return int(kept.value)

    def _check_utf8(self, rows: int):
        """The names of the last `rows` queued rows decoded as the host reader decodes them: the first one that is not
        valid UTF-8 raises the decoder's own UnicodeDecodeError."""
        buf, n = C.create_string_buffer(1 << 16), C.c_int64()
        while True:
            rc = self.lib.c2v_reader_eval_check_utf8(self.h, rows, buf, len(buf), C.byref(n), self.stream.cuda_stream)
            if rc != 0:
                raise EngineError(rc, self.lib.c2v_last_error(None).decode())
            if n.value <= len(buf):
                break
            buf = C.create_string_buffer(n.value)          # a name longer than the buffer: again, all of it
        if n.value >= 0:
            name = buf.raw[:n.value]
            name.decode("utf-8")
            raise RuntimeError("c2v_reader_eval_check_utf8 flagged a name the UTF-8 decoder accepts: %r" % name)

    def eval_words(self):
        """(words, word_off, n_words): the device pointers of the target words of an evaluation reader's tables."""
        w, off, n = C.c_void_p(), C.c_void_p(), C.c_int32()
        rc = self.lib.c2v_reader_eval_words(self.h, C.byref(w), C.byref(off), C.byref(n))
        if rc != 0:
            raise EngineError(rc, self.lib.c2v_last_error(None).decode())
        return w.value, off.value, int(n.value)

    def _take(self, b: int, k: int):
        """Batch k: the queue's next b rows and their names; None when the consumer has gone."""
        s = self._acquire(k)
        if s is None:
            return None
        if s["names"].numel() < self._name_bytes:          # the slot's last reader is done (_acquire): it may grow
            s["names"] = self.torch.empty(max(self._name_bytes, 2 * s["names"].numel()), dtype=self.torch.uint8,
                                          device=self.dev)
        t = s["tensors"]
        rc = self.lib.c2v_reader_eval_take(self.h, b, *(x.data_ptr() for x in t), s["name_off"].data_ptr(),
                                           s["names"].data_ptr(), s["names"].numel(), self.stream.cuda_stream)
        if rc != 0:
            raise EngineError(rc, self.lib.c2v_last_error(None).decode())
        s["ready"].record(self.stream)
        return DeviceBatch(s, b, 0, b, 0, self)

    def _run_eval(self, put) -> bool:
        """One pass over the test file: every batch is the queue's next B rows, the last one what remains.  False when
        the consumer has gone."""
        n, k = 0, 0
        chunks = self.reader._native_chunks_ahead()
        try:
            for i, chunk in enumerate(chunks):
                n += self._append(chunk, i % 2)
                while n >= self.B:
                    batch = self._take(self.B, k)
                    if batch is None or not put(batch):
                        return False
                    n, k = n - self.B, k + 1
        finally:
            chunks.close()
        if n > 0:
            batch = self._take(n, k)
            if batch is None or not put(batch):
                return False
        return True

    def score(self, batch: "DeviceBatch", ids) -> EvalScores:
        """The metric kernel (c2v_reader_eval_score) on the top-k ids [rows, k] (int32, device) of an evaluation batch,
        queued on the current stream; then the per-row results, the accumulators and the names are copied to the host
        (the current stream is synchronised).  The ids come back too when a row is flagged."""
        torch = self.torch
        s = batch._slot
        n, k = batch.hi - batch.lo, int(ids.shape[1])
        r = s.get("res")
        if r is None or r["acc"].numel() != k + 4:
            r = {"rff": torch.empty((3, self.B), dtype=torch.int32, device=self.dev),
                 "acc": torch.empty(k + 4, dtype=torch.int64, device=self.dev),
                 "h_rff": torch.empty((3, self.B), dtype=torch.int32).pin_memory(),
                 "h_acc": torch.empty(k + 4, dtype=torch.int64).pin_memory(),
                 "h_off": torch.empty(self.B + 1, dtype=torch.int64).pin_memory()}
            s["res"] = r
        st = torch.cuda.current_stream(self.dev)
        rff = r["rff"]
        rc = self.lib.c2v_reader_eval_score(self.h, ids.data_ptr(), n, k, s["name_off"].data_ptr(), s["names"].data_ptr(),
                                            rff[0].data_ptr(), rff[1].data_ptr(), rff[2].data_ptr(), r["acc"].data_ptr(),
                                            st.cuda_stream)
        if rc != 0:
            raise EngineError(rc, self.lib.c2v_last_error(None).decode())
        r["h_rff"][:, :n].copy_(rff[:, :n], non_blocking=True)
        r["h_acc"].copy_(r["acc"], non_blocking=True)
        r["h_off"][:n + 1].copy_(s["name_off"][:n + 1], non_blocking=True)
        st.synchronize()
        rff_h = r["h_rff"][:, :n].numpy().copy()
        off = r["h_off"][:n + 1].numpy().copy()
        names = s["names"][:int(off[n])].cpu().numpy().tobytes()
        flagged = bool(rff_h[2].any())
        return EvalScores(rff_h[0], rff_h[1], rff_h[2], r["h_acc"].numpy().copy(), (names, off),
                          ids[:n].cpu().numpy() if flagged else None)

    # ---- sharded chunks ----------------------------------------------------------------------------------------------
    def _stage(self, j: int, rows: int):
        """This rank's stage j with room for `rows` rows, and its handle if it is new (None otherwise)."""
        s = self._stages[j]
        if s is not None and s["rows"] >= rows:
            return s, None
        if s is not None:
            # the peers close the old stage when the new handle reaches them in the coming exchange, before they enter
            # the one after it: once that one is over, nobody has it open
            self._retired.append((s["ptr"], self._exchanges + 2))
            rows = max(rows, s["rows"] * 5 // 4)
        nbytes = int(self.lib.c2v_reader_stage_bytes(self.C, rows))
        ptr, handle = self.transport.alloc(nbytes)
        # c2v_ipc_alloc zero-fills the new stage with a cudaMemset on the legacy default stream, which returns before the
        # fill has run and which the reader stream (non-blocking) is not ordered after.  The parse that writes the stage
        # must not run before the fill, or the fill, queued behind the training steps on that stream, could land later
        # and zero rows, keep flags and the status header that the owner and its peers then read at different times.
        filled = self.torch.cuda.Event()
        filled.record(self.torch.cuda.default_stream(self.dev))
        self.stream.wait_event(filled)
        self._stages[j] = s = {"ptr": ptr, "rows": rows, "bytes": nbytes}
        return s, handle

    def _exchange(self, msg) -> list:
        got = self.transport.gather(msg)
        self._exchanges += 1
        for ptr, due in [x for x in self._retired if x[1] <= self._exchanges]:
            self.transport.free(ptr)
            self._retired.remove((ptr, due))
        return got

    def _raise_if_a_peer_failed(self, got):
        """Raises when a message of an exchange (status, handle, error) carries a rank's error: every rank raises."""
        failed = [(r, m[2]) for r, m in enumerate(got) if m is not None and m[2]]
        if failed:
            self._peers_know = True
            raise RuntimeError("rank %d of the sharded device reader failed: %s" % failed[0])

    def _leave(self, why: str):
        """This rank stops reading before the pass is over (an error after an exchange, or its consumer stopped): its
        peers learn it in the exchange they enter next, and raise, instead of waiting for it there.  Nothing to do when
        the peers know already (the error came out of an exchange, or the last exchange of the pass is behind)."""
        if self.transport is None or self._peers_know:
            return
        self._peers_know = True
        try:
            self._exchange((None, None, why))
        except Exception:                              # the peers may have gone too; the rank's own error stands
            pass

    def _parse_sharded(self, fd: int, a: int, b: int, k: int) -> int:
        """Chunk k = [a, b) of file fd: this rank's share read, uploaded and parsed into stage k % 2, the shares' statuses
        exchanged, then every stage assembled into the pool in rank order and committed.  Returns the rows kept."""
        torch, j = self.torch, k % 2
        status = handle = err = None
        try:
            s0, s1 = share_range(fd, a, b, self.world, self.rank)
            n = s1 - s0
            # Stage j last held chunk k - 2.  Every peer finished assembling that chunk (commit_shares synchronises)
            # before it entered the exchange of chunk k - 1, which this rank has left, so no peer reads stage j now: it
            # may be overwritten, grown or replaced.
            stage, handle = self._stage(j, n // (self.C + 1) + 1)
            text = 0
            if n:
                buf = self._text_buffers(j, n)
                buf["uploaded"].synchronize()                   # the previous upload out of this host buffer has left
                pread_into(fd, buf["np"][:n], s0)
                with torch.cuda.stream(self.copy_stream):
                    buf["dev"][:n].copy_(buf["host"][:n], non_blocking=True)
                    buf["uploaded"].record(self.copy_stream)
                self.stream.wait_event(buf["uploaded"])
                self.h2d_bytes += n
                text = buf["dev"].data_ptr()
            st = c2v_reader_share_status()
            rc = self.lib.c2v_reader_parse_share(self.h, text, n, b - a, stage["ptr"], stage["rows"], C.byref(st),
                                                 self.stream.cuda_stream)          # synchronises: the stage is complete
            if rc != 0:
                raise EngineError(rc, self.lib.c2v_last_error(None).decode())
            status = tuple(getattr(st, f) for f, _ in st._fields_)
        except Exception as exc:
            err = exc
        # every rank enters the exchange, a failed one too, so that none waits for a rank that has gone
        got = self._exchange((status, handle, None if err is None else "%s: %s" % (type(err).__name__, err)))
        if err is not None:
            self._peers_know = True
            raise err
        self._raise_if_a_peer_failed(got)
        statuses = [c2v_reader_share_status(*m[0]) for m in got]
        bad = chunk_error(statuses, b - a, self.C)
        if bad is not None:
            self._peers_know = True                    # every rank decides the same error from the same statuses
            raise_chunk_error(bad, self.C)
        for r, m in enumerate(got):
            if r != self.rank and m[1] is not None:
                old = self._peers.pop((r, j), None)
                if old is not None:
                    self.transport.close(old)
                self._peers[(r, j)] = self.transport.open(m[1])
        W = self.world
        ptrs = (C.c_void_p * W)(*[self._stages[j]["ptr"] if r == self.rank else self._peers[(r, j)] for r in range(W)])
        recs = (C.c_int64 * W)(*[s.records for s in statuses])
        kept = C.c_int64()
        rc = self.lib.c2v_reader_commit_shares(self.h, ptrs, recs, W, C.byref(kept), self.stream.cuda_stream)
        if rc != 0:
            raise EngineError(rc, self.lib.c2v_last_error(None).decode())
        self.peer_bytes += sum(s.records for r, s in enumerate(statuses) if r != self.rank) * self._row_bytes
        return int(kept.value)

    def _acquire(self, k: int):
        s = self.slots[k % len(self.slots)]
        while not s["free"].wait(timeout=0.1):
            if self._stop.is_set():
                return None
        s["done"].synchronize()                             # the step that last read this slot has run
        s["free"].clear()
        return s

    def _draw(self, n: int, b: int, k: int):
        """Batch k: b of the n pool rows, drawn as _RowPool.take draws them; None when the consumer has gone."""
        s = self._acquire(k)
        if s is None:
            return None
        pick = self.reader._rng.choice(n, size=b, replace=False) if b < n else self.reader._rng.permutation(n)
        host = s["pick"].numpy()
        host[:b] = pick
        lo, hi, dropped = batch_split(b, self.world, self.rank) if self.world > 1 else (0, b, 0)
        t = s["tensors"]
        self.h2d_bytes += 8 * b
        rc = self.lib.c2v_reader_draw(self.h, host.ctypes.data, b, lo, hi, *(x.data_ptr() for x in t),
                                      self.stream.cuda_stream)
        if rc != 0:
            raise EngineError(rc, self.lib.c2v_last_error(None).decode())
        s["ready"].record(self.stream)
        return DeviceBatch(s, b, lo, hi, dropped, self)

    def _run(self, q: "queue.Queue", done):
        def put(item) -> bool:
            while not self._stop.is_set():
                try:
                    q.put(item, timeout=0.1)
                    return True
                except queue.Full:
                    continue
            return False

        try:
            with self.torch.cuda.device(self.dev):
                if self.evaluate:
                    if self._run_eval(put):
                        put(done)
                    return
                n, k = 0, 0
                if self.transport is not None:
                    chunks = self.reader._native_chunk_ranges()
                    parse = lambda chunk, i: self._parse_sharded(*chunk, i)
                else:
                    chunks = self.reader._native_chunks_ahead()
                    parse = lambda chunk, i: self._parse(chunk, i % 2)
                try:
                    for i, chunk in enumerate(chunks):
                        n += parse(chunk, i)
                        while n >= self.S + self.B:
                            batch = self._draw(n, self.B, k)
                            if batch is None or not put(batch):
                                self._leave("rank %d stopped reading: its consumer has gone" % self.rank)
                                return
                            n, k = n - self.B, k + 1
                finally:
                    chunks.close()
                if self.transport is not None:
                    # every rank has assembled the last chunk: no stage is read any more
                    got = self._exchange(None)
                    self._peers_know = True
                    self._raise_if_a_peer_failed(got)
                while n > 0:
                    b = min(self.B, n)
                    batch = self._draw(n, b, k)
                    if batch is None or not put(batch):
                        return
                    n, k = n - b, k + 1
            put(done)
        except BaseException as exc:
            self._leave("rank %d failed: %s: %s" % (self.rank, type(exc).__name__, exc))
            put(exc)

    def __iter__(self):
        if self._thread is not None and self.evaluate and not self._thread.is_alive():
            # an evaluation reader reads the test file again: its queue is empty once a pass has ended
            self._thread.join()
            if self.lib.c2v_reader_eval_queued(self.h) != 0:
                raise RuntimeError("the last evaluation pass stopped early; make a new DeviceBatchReader")
            self._thread = None
            self._stop.clear()
        if self._thread is not None:
            raise RuntimeError("a DeviceBatchReader reads one pass; make a new one for the next")
        q: "queue.Queue" = queue.Queue(maxsize=len(self.slots))
        done = object()
        self._thread = threading.Thread(target=self._run, args=(q, done), daemon=True)
        self._thread.start()
        try:
            while True:
                item = q.get()
                if item is done:
                    return
                if isinstance(item, BaseException):
                    raise item
                yield item
        finally:
            self._stop.set()

    # ---- life cycle --------------------------------------------------------------------------------------------------
    def device_bytes(self) -> int:
        """Device memory the reader holds: vocabularies (shared with the model's other reader when given), batch slots
        (with an evaluation batch's names and results), chunk text, this rank's stages (sharded) and the handle's pool,
        scratch, evaluation queue and tables."""
        n = self.vocabs.nbytes()
        n += sum(t.numel() * t.element_size() for s in self.slots for t in s["tensors"])
        n += sum(t.numel() * t.element_size() for s in self.slots for key in ("name_off", "names") if key in s
                 for t in (s[key],))
        n += sum(t.numel() * t.element_size() for s in self.slots if "res" in s for key in ("rff", "acc")
                 for t in (s["res"][key],))
        n += sum(b["dev"].numel() for b in self._text if b is not None)
        n += sum(s["bytes"] for s in self._stages if s is not None)
        return int(n + (self.lib.c2v_reader_device_bytes(self.h) if self.h else 0))

    def close(self):
        """Stops the reader thread and frees what the reader holds.  A sharded reader's stages are freed here: after a
        whole pass every peer is done with them; after a failed one the peers stopped at the same exchange."""
        self._stop.set()
        if self._thread is not None:
            self._thread.join()
        if getattr(self, "h", None):
            self.lib.c2v_reader_destroy(self.h)        # synchronises the device first
            self.h = None
        if self.transport is not None:
            for ptr in self._peers.values():
                self.transport.close(ptr)
            self._peers = {}
            for ptr in [s["ptr"] for s in self._stages if s is not None] + [p for p, _ in self._retired]:
                self.transport.free(ptr)
            self._stages, self._retired = [None, None], []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
