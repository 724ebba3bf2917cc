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
indices (8 bytes a row).  Code2VecModel.train() uses it when C2V_DEVICE_READER=1."""
from __future__ import annotations

import ctypes as C
import queue
import threading
from typing import Optional

import numpy as np

from .engine import EngineError, c2v_reader_vocab, load_library
from .multi_rank import batch_split
from .path_context_reader import _INT64_MIN, PathContextReader, _raise_parse_error


def device_reader_flag(environ) -> bool:
    """C2V_DEVICE_READER=1: Code2VecModel.train() reads its batches on the GPU; 0 (the default): on the host."""
    flag = environ.get("C2V_DEVICE_READER", "0") or "0"
    if flag not in ("0", "1"):
        raise ValueError("C2V_DEVICE_READER must be 0 or 1, got %r" % flag)
    return flag == "1"


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


class DeviceBatch:
    """One batch in a device slot: `tensors` = (src, path, tgt [rows, C] int32, mask [rows, C] float32, target [rows]
    int32) holding rows [lo, hi) of a global batch of `rows` rows (all of it on one GPU); `dropped` rows of a short batch
    are left out on several ranks (multi_rank.batch_split).  wait() makes the current stream wait for the draw; release()
    hands the slot back once the work queued so far on the current stream (the step that read it) is done."""
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
    use_native=True does)."""

    def __init__(self, reader: PathContextReader, device, world: int = 1, rank: int = 0, slots: int = 4):
        import torch
        if not reader.estimator_action.is_train:
            raise ValueError("the device reader reads training files only")
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
        self.B = int(cfg.TRAIN_BATCH_SIZE)
        self.S = max(int(cfg.SHUFFLE_BUFFER_SIZE), 1)
        self.h2d_bytes = 0
        lib_b, tok, pth, tgt = reader._native
        self._vocab_tensors = []
        structs = []
        with torch.cuda.device(self.dev):
            for v in (tok, pth, tgt):
                slot_arr, byte_arr, mask, oov, pad = export_vocab(lib_b, v.h)
                d_slots = torch.from_numpy(slot_arr).to(self.dev)
                d_bytes = torch.from_numpy(byte_arr if byte_arr.size else np.zeros(1, dtype=np.uint8)).to(self.dev)
                self._vocab_tensors += [d_slots, d_bytes]
                structs.append(c2v_reader_vocab(d_slots.data_ptr(), d_bytes.data_ptr(), mask, oov, pad))
            torch.cuda.synchronize(self.dev)
            h = C.c_void_p()
            rc = self.lib.c2v_reader_create(self.C, C.byref(structs[0]), C.byref(structs[1]), C.byref(structs[2]),
                                            self.dev.index or 0, C.byref(h))
            if rc != 0:
                raise EngineError(rc, self.lib.c2v_last_error(None).decode())
            self.h = h
            self.stream = torch.cuda.Stream(device=self.dev)
            self.copy_stream = torch.cuda.Stream(device=self.dev)
            local = self.B // self.world
            self.slots = []
            for _ in range(slots):
                s = {"tensors": (torch.empty((local, self.C), dtype=torch.int32, device=self.dev),
                                 torch.empty((local, self.C), dtype=torch.int32, device=self.dev),
                                 torch.empty((local, self.C), dtype=torch.int32, device=self.dev),
                                 torch.empty((local, self.C), dtype=torch.float32, device=self.dev),
                                 torch.empty((local,), dtype=torch.int32, device=self.dev)),
                     "pick": torch.empty(self.B, dtype=torch.int64).pin_memory(),
                     "ready": torch.cuda.Event(), "done": torch.cuda.Event(), "free": threading.Event()}
                s["free"].set()
                self.slots.append(s)
        # chunk text: two page-locked buffers and two device buffers, so the upload of chunk k+1 overlaps the draws of k
        self._text = [None, None]
        self._thread: Optional[threading.Thread] = None
        self._stop = threading.Event()

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
                n, k = 0, 0
                chunks = self.reader._native_chunks_ahead()
                try:
                    for i, chunk in enumerate(chunks):
                        n += self._parse(chunk, i % 2)
                        while n >= self.S + self.B:
                            batch = self._draw(n, self.B, k)
                            if batch is None or not put(batch):
                                return
                            n, k = n - self.B, k + 1
                finally:
                    chunks.close()
                while n > 0:
                    b = min(self.B, n)
                    batch = self._draw(n, b, k)
                    if batch is None or not put(batch):
                        return
                    n, k = n - b, k + 1
            put(done)
        except BaseException as exc:
            put(exc)

    def __iter__(self):
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
        """Device memory the reader holds: vocabularies, batch slots, chunk text and the handle's pool and scratch."""
        n = sum(t.numel() * t.element_size() for t in self._vocab_tensors)
        n += sum(t.numel() * t.element_size() for s in self.slots for t in s["tensors"])
        n += sum(b["dev"].numel() for b in self._text if b is not None)
        return int(n + (self.lib.c2v_reader_device_bytes(self.h) if self.h else 0))

    def close(self):
        self._stop.set()
        if self._thread is not None:
            self._thread.join()
        if getattr(self, "h", None):
            self.lib.c2v_reader_destroy(self.h)        # synchronises the device first
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
