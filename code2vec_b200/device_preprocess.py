"""Dataset preparation on the GPU (DESIGN.md §6g): preprocess.main's command line with the text work in device memory.

The raw files are read in chunks of whole lines (chunk_ranges: universal newlines, as open(path, "r") reads them), each
chunk is copied into a page-locked buffer and uploaded, and the kernels of libc2v_b200.so (include/c2v_b200.h,
"Preprocessing on the device") check it as UTF-8, index its lines and
  * count the histograms (count_histograms): one device hash table of every token, path and target with its count and
    the offset of its first occurrence, written out in first-occurrence order -- Counter's insertion order;
  * down-sample each file (process_file): the device classifies the contexts of every line longer than max_contexts
    and reports (n_full, n_partial) per such line; the host draws rng.sample(range(n), k) on the caller's own rng for
    exactly the lines the host route samples, in file order (random.sample consumes the stream through len(population)
    and k only, and returns the indices rng.sample(list, k) would pick), and the device writes the output lines in the
    order of those picks.  A chunk's text reaches the file only once the next chunk's copy is queued.
Vocabulary cut-offs (load_histogram) and the `.dict.c2v` pickles are the host's code; the vocabularies go to the device
as the native tensoriser's hash tables (c2v_vocab_create / c2v_vocab_export).  The files, the log lines of process_file
and the state the rng is left in are those of the host route.  preprocess.main uses it when C2V_DEVICE_PREPROCESS=1."""
from __future__ import annotations

import ctypes as C
import os
import time
from typing import Callable, Iterable, Iterator, Optional, Tuple

import numpy as np

from . import preprocess as P

WINDOW_BYTES = 32 << 20        # a chunk's window: cut after its last line end (doubled while it holds none)
_SCAN_BYTES = 1 << 16          # the backward scan for a window's last line end reads this many bytes at a time
_KINDS = {"word": 0, "path": 1, "target": 2}


def device_preprocess_flag(environ) -> bool:
    """C2V_DEVICE_PREPROCESS=1: preprocess.main runs on the GPU; 0 (the default): on the host."""
    flag = environ.get("C2V_DEVICE_PREPROCESS", "0") or "0"
    if flag not in ("0", "1"):
        raise ValueError("C2V_DEVICE_PREPROCESS must be 0 or 1, got %r" % flag)
    return flag == "1"


# ---- chunks of whole lines -------------------------------------------------------------------------------------------
def last_line_end(read: Callable[[int, int], bytes], lo: int, hi: int, size: int) -> int:
    """The largest q in (lo, hi] at which a line of the file ends -- byte q - 1 is '\\n', or '\\r' not followed by
    '\\n' -- or -1.  read(offset, n) returns the file's bytes; the byte after hi is read too, as a '\\r' at hi - 1 ends
    no line when a '\\n' follows it."""
    while hi > lo:
        a = max(lo, hi - _SCAN_BYTES)
        blk = read(a, min(hi + 1, size) - a)
        n = hi - a
        i = blk.rfind(b"\n", 0, n)
        j = blk.rfind(b"\r", i + 1, n)
        if j >= 0 and j + 1 < len(blk) and blk[j + 1] == 0x0A:
            j = blk.rfind(b"\r", i + 1, j)
        k = max(i, j)
        if k >= 0:
            return a + k + 1
        hi = a
    return -1


def chunk_ranges(read: Callable[[int, int], bytes], size: int, window: int) -> Iterator[Tuple[int, int]]:
    """The chunks [a, b) of a file of `size` bytes: a window from the previous chunk's end is cut after its last line
    end; a window with none (a line longer than it) is retried twice as large, and the larger window stays; the window
    that reaches the end of the file is the last chunk whole."""
    start, w = 0, int(window)
    while start < size:
        if size - start <= w:
            yield start, size
            return
        cut = last_line_end(read, start, start + w, size)
        if cut < 0:
            w *= 2
            continue
        yield start, cut
        start = cut


def line_spans(text: bytes):
    """(start, end) of every line of a chunk, end excluding its terminator: the line index the device computes."""
    starts = [p for p in range(len(text))
              if p == 0 or text[p - 1] == 0x0A or (text[p - 1] == 0x0D and text[p] != 0x0A)]
    spans = []
    for i, s in enumerate(starts):
        e = starts[i + 1] if i + 1 < len(starts) else len(text)
        while e > s and text[e - 1] in (0x0A, 0x0D):
            e -= 1
        spans.append((s, e))
    return spans


# ---- the device route ------------------------------------------------------------------------------------------------
class DevicePreprocessor:
    """One preprocessing run's device state on `device`: a c2v_prep handle, the text buffers and the membership tables.
    close() frees them."""

    def __init__(self, device=0, window: int = WINDOW_BYTES):
        import torch
        from .engine import EngineError, load_library
        self.torch, self.EngineError = torch, EngineError
        self.lib = load_library()
        self.dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        self.window = int(window)
        self.stream = torch.cuda.Stream(self.dev)
        self.h = C.c_void_p()
        self._check(self.lib.c2v_prep_create(self.dev.index or 0, C.byref(self.h)))
        self._in_host = self._in_dev = None
        self._out = [None, None]                    # page-locked copies of the output text, one per pending chunk
        self._events = [torch.cuda.Event(), torch.cuda.Event()]
        self._vocabs = None
        self.uploaded = 0
        self.peak_device_bytes = self.peak_host_bytes = 0
        self.phase_s = {"read": 0.0, "count": 0.0, "classify": 0.0, "sample": 0.0, "assemble": 0.0, "write": 0.0}

    def _check(self, rc):
        if rc != 0:
            raise self.EngineError(rc, self.lib.c2v_last_error(None).decode())

    def _peaks(self):
        held = lambda t: 0 if t is None else t.numel() * t.element_size()
        dev = int(self.lib.c2v_prep_device_bytes(self.h)) + held(self._in_dev) + (self._vocabs.nbytes if self._vocabs else 0)
        host = held(self._in_host) + sum(held(t) for t in self._out)
        self.peak_device_bytes = max(self.peak_device_bytes, dev)
        self.peak_host_bytes = max(self.peak_host_bytes, host)

    def close(self):
        if self.h:
            self.lib.c2v_prep_destroy(self.h)
            self.h = C.c_void_p()
        self._in_host = self._in_dev = self._vocabs = None
        self._out = [None, None]

    # ---- input -------------------------------------------------------------------------------------------------------
    def _chunks(self, path: str):
        """(file offset, device pointer, bytes) of every chunk of the file, uploaded on the handle's stream."""
        torch = self.torch
        with open(path, "rb") as f:
            fd = f.fileno()
            size = os.fstat(fd).st_size
            read = lambda off, n: os.pread(fd, n, off)
            for a, b in chunk_ranges(read, size, self.window):
                n = b - a
                t0 = time.perf_counter()
                if self._in_host is None or self._in_host.numel() < n:
                    self.stream.synchronize()
                    self._in_host = None
                    self._in_dev = None
                    self._in_host = torch.empty(max(n, 1), dtype=torch.uint8, pin_memory=True)
                    self._in_dev = torch.empty(max(n, 1), dtype=torch.uint8, device=self.dev)
                from .path_context_reader import pread_into
                pread_into(fd, self._in_host[:n].numpy(), a)
                with torch.cuda.stream(self.stream):
                    self._in_dev[:n].copy_(self._in_host[:n], non_blocking=True)
                self.uploaded += n
                self.phase_s["read"] += time.perf_counter() - t0
                self._peaks()
                yield a, self._in_dev.data_ptr(), n

    def _utf8_error(self, path: str, offset: int):
        with open(path, "rb") as f:
            f.seek(offset)
            bad = f.read(4)
        return UnicodeDecodeError("utf-8", bad, 0, 1, "invalid UTF-8 at byte %d of %s" % (offset, path))

    # ---- count_histograms --------------------------------------------------------------------------------------------
    def count_histograms(self, train_path: str) -> Tuple[int, int, int]:
        """Counts the tokens, paths and targets of the raw training file into the handle's table."""
        st = self._status()
        for a, ptr, n in self._chunks(train_path):
            t0 = time.perf_counter()
            self._check(self.lib.c2v_prep_count_chunk(self.h, ptr, n, a, C.byref(st), self.stream.cuda_stream))
            self.phase_s["count"] += time.perf_counter() - t0
            if st.bad_utf8 >= 0:
                raise self._utf8_error(train_path, a + st.bad_utf8)
        self._peaks()
        self.table = (int(st.keys), int(st.slots), int(st.rehashes))
        return self.table

    def write_histogram(self, kind: str, path: str):
        """write_histogram's file of the counted `kind` ("word", "path" or "target")."""
        t0 = time.perf_counter()
        ptr, n = C.c_void_p(), C.c_int64()
        self._check(self.lib.c2v_prep_histogram(self.h, _KINDS[kind], C.byref(ptr), C.byref(n), self.stream.cuda_stream))
        buf = self.torch.empty(max(n.value, 1), dtype=self.torch.uint8, pin_memory=True)
        if n.value:
            with self.torch.cuda.stream(self.stream):
                buf[:n.value].copy_(self._device_view(ptr.value, n.value), non_blocking=True)
        self.stream.synchronize()
        with open(path, "wb") as f:
            f.write(memoryview(buf.numpy())[:n.value])
        self.phase_s["count"] += time.perf_counter() - t0
        self._peaks()

    # ---- process_file ------------------------------------------------------------------------------------------------
    def set_vocabularies(self, word_to_count, path_to_count):
        """Membership tables of the two vocabularies on the device."""
        self._vocabs = _MembershipTables(self.dev, (word_to_count, path_to_count))

    @staticmethod
    def _status():
        from .engine import c2v_prep_status
        return c2v_prep_status()

    def process_file(self, file_path: str, data_file_role: str, dataset_name: str, max_contexts: int, rng,
                     log=print) -> int:
        """preprocess.process_file on the device: the same file, log lines and rng draws."""
        torch = self.torch
        C_ = int(max_contexts)
        if C_ < 0:
            raise ValueError("max_contexts must be >= 0, got %d" % C_)
        sample = rng.sample
        seen = kept = written = empty = longest = 0
        line0 = 0
        st = self._status()
        tok, pth = self._vocabs.structs
        pending = None
        slot = 0
        with open("%s.%s.c2v" % (dataset_name, data_file_role), "wb") as out:
            for a, ptr, n in self._chunks(file_path):
                t0 = time.perf_counter()
                self._check(self.lib.c2v_prep_classify_chunk(self.h, ptr, n, C_, C.byref(tok), C.byref(pth), C.byref(st),
                                                             self.stream.cuda_stream))
                if st.bad_utf8 >= 0:
                    raise self._utf8_error(file_path, a + st.bad_utf8)
                nl = int(st.long_lines)
                lines = np.empty(nl, dtype=np.int64)
                nf = np.empty(nl, dtype=np.int32)
                npart = np.empty(nl, dtype=np.int32)
                self._check(self.lib.c2v_prep_long_lines(self.h, lines.ctypes.data, nf.ctypes.data, npart.ctypes.data,
                                                         self.stream.cuda_stream))
                t1 = time.perf_counter()
                self.phase_s["classify"] += t1 - t0
                # the host's draws, in file order, for the lines the host samples (up to a line that raises)
                stop = nl if st.bad_line < 0 else int(np.searchsorted(lines, st.bad_line))
                picks, off = [], np.zeros(nl + 1, dtype=np.int64)
                extend = picks.extend
                for r, (f, p) in enumerate(zip(nf[:stop].tolist(), npart[:stop].tolist())):
                    if f > C_:
                        extend(sample(range(f), C_))
                    elif f + p > C_:
                        extend(sample(range(p), C_ - f))
                    off[r + 1] = len(picks)
                t2 = time.perf_counter()
                self.phase_s["sample"] += t2 - t1
                if st.bad_line >= 0:
                    raise IndexError("list index out of range: line %d of %s has more than %d contexts and one of "
                                     "fewer than 3 comma-separated parts" % (line0 + st.bad_line + 1, file_path, C_))
                pk = np.asarray(picks, dtype=np.int32)
                ptr_out, nbytes = C.c_void_p(), C.c_int64()
                self._check(self.lib.c2v_prep_assemble(self.h, pk.ctypes.data if pk.size else None, off.ctypes.data,
                                                       C.byref(ptr_out), C.byref(nbytes), self.stream.cuda_stream))
                nb = int(nbytes.value)
                buf = self._out[slot]
                if buf is None or buf.numel() < nb:
                    self._out[slot] = None
                    self._out[slot] = buf = torch.empty(max(nb, 1), dtype=torch.uint8, pin_memory=True)
                if nb:
                    with torch.cuda.stream(self.stream):
                        buf[:nb].copy_(self._device_view(ptr_out.value, nb), non_blocking=True)
                self._events[slot].record(self.stream)
                self.phase_s["assemble"] += time.perf_counter() - t2
                self._peaks()
                self._flush(out, pending)          # the previous chunk's text, now that this one is queued
                pending = (slot, nb)
                slot ^= 1
                seen += st.seen
                kept += st.kept
                written += st.written
                empty += st.empty
                longest = max(longest, int(st.longest))
                line0 += st.lines
            self._flush(out, pending)
        P.log_file_stats(file_path, seen, kept, written, empty, longest, log)
        return written

    def _device_view(self, ptr: int, n: int):
        """A uint8 tensor over n bytes of the handle's device memory at ptr."""
        arr = type("DeviceBytes", (), {"__cuda_array_interface__": {
            "shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 2, "strides": None,
            "stream": None}})()
        return self.torch.as_tensor(arr, device=self.dev)

    def _flush(self, out, pending):
        if pending is None:
            return
        t0 = time.perf_counter()
        s, nb = pending
        self._events[s].synchronize()
        out.write(memoryview(self._out[s].numpy())[:nb])
        self.phase_s["write"] += time.perf_counter() - t0

    def report(self) -> str:
        return ("%.1f MB of text uploaded; %.1f MB of device memory and %.1f MB of page-locked host memory held at most"
                % (self.uploaded / 1e6, self.peak_device_bytes / 1e6, self.peak_host_bytes / 1e6))


class _MembershipTables:
    """The word and path vocabularies as the native tensoriser's hash tables (c2v_vocab_create, every word index 1, oov
    0), copied to the device, with the c2v_reader_vocab structs that point at them."""

    def __init__(self, dev, vocabs):
        import torch
        from .device_reader import export_vocab
        from .engine import c2v_reader_vocab
        from .path_context_reader import load_native_tensoriser
        lib = load_native_tensoriser()
        if lib is None:
            raise RuntimeError("the device route needs libc2v_batcher.so (code2vec_b200/native/build_native.py)")
        self.tensors, self.structs = [], []
        self.nbytes = 0
        for words in vocabs:
            enc = [w.encode("utf-8") for w in words]
            offsets = np.zeros(len(enc) + 1, dtype=np.int64)
            np.cumsum([len(b) for b in enc], out=offsets[1:])
            idx = np.ones(len(enc), dtype=np.int32)
            h = lib.c2v_vocab_create(b"".join(enc), offsets.ctypes.data, idx.ctypes.data, len(enc), 0, 0)
            try:
                slot_arr, byte_arr, mask, oov, pad = export_vocab(lib, h)
                d_slots = torch.from_numpy(slot_arr.copy()).to(dev)
                d_bytes = torch.from_numpy(byte_arr.copy() if byte_arr.size else np.zeros(1, dtype=np.uint8)).to(dev)
            finally:
                lib.c2v_vocab_destroy(h)
            self.tensors += [d_slots, d_bytes]
            self.nbytes += d_slots.numel() + d_bytes.numel()
            self.structs.append(c2v_reader_vocab(d_slots.data_ptr(), d_bytes.data_ptr(), mask, oov, pad))
        torch.cuda.synchronize(dev)


def main(argv: Optional[Iterable[str]] = None, rng=None, log=print, device=0, window: int = WINDOW_BYTES,
         stats: Optional[dict] = None) -> int:
    """preprocess.main with the histograms and the `.c2v` files made on the GPU.  `stats`, when given, receives the
    seconds of each phase and the memory report."""
    import random
    rng = random if rng is None else rng
    args = P.arguments_parser().parse_args(None if argv is None else list(argv))
    prep = DevicePreprocessor(device, window)
    log("Preprocessing on the GPU (C2V_DEVICE_PREPROCESS=1): %s" % prep.dev)
    try:
        histos = {"word": args.word_histogram, "path": args.path_histogram, "target": args.target_histogram}
        if not all(histos.values()):
            prep.count_histograms(args.train_data_path)
            for kind, given in histos.items():
                if not given:
                    histos[kind] = "%s.histo.%s.c2v" % (args.output_name, {"word": "ori", "path": "path", "target": "tgt"}[kind])
                    prep.write_histogram(kind, histos[kind])
        word_to_count = P.load_histogram(histos["word"], int(args.word_vocab_size))
        path_to_count = P.load_histogram(histos["path"], int(args.path_vocab_size))
        target_to_count = P.load_histogram(histos["target"], int(args.target_vocab_size))
        prep.set_vocabularies(word_to_count, path_to_count)
        num_training_examples = 0
        for file_path, role in ((args.test_data_path, "test"), (args.val_data_path, "val"), (args.train_data_path, "train")):
            n = prep.process_file(file_path, role, args.output_name, int(args.max_contexts), rng, log)
            if role == "train":
                num_training_examples = n
        P.save_dictionaries(args.output_name, word_to_count, path_to_count, target_to_count, num_training_examples, log)
        log("Device preprocessing: " + prep.report())
        if stats is not None:
            stats.update(phases_s=dict(prep.phase_s), report=prep.report(), table=getattr(prep, "table", None))
    finally:
        prep.close()
    return num_training_examples
