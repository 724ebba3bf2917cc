"""`.vectors` and word2vec files formatted on the GPU (DESIGN.md §6f).

The host writers (model_base._write_code_vectors, common.save_word2vec_file) turn every float32 into text with one
Python str() each.  DeviceTextWriter hands the rows of a float32 matrix in device memory to c2v_text_format_rows
(include/c2v_b200.h, "Text of float32 matrices"), which writes numpy's str() of every value on the device, and writes
the text it brings back to a binary file: the same bytes, in bounded chunks.
  * A chunk is as many rows as fit `chunk_bytes` (64 MB) at the text's bound of C2V_TEXT_VALUE_BYTES per value plus the
    row's prefix, so even the 1.3 M-row token table of java14m needs no more text buffer than that.
  * Each chunk's text is copied into one of two page-locked buffers.  The text of a chunk is written to the file with one
    write() once the next chunk's format and copy are queued, so the GPU works on chunk k + 1 while the host writes
    chunk k -- also across write_rows calls, as evaluate() makes one per batch.
Code2VecModel uses it when C2V_DEVICE_TEXT=1."""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

from .engine import EngineError, load_library

CHUNK_BYTES = 64 << 20
VALUE_BYTES = 16          # C2V_TEXT_VALUE_BYTES: one value's text (at most 15 bytes) and its separator


def device_text_flag(environ) -> bool:
    """C2V_DEVICE_TEXT=1: `.vectors` and word2vec files are formatted on the GPU; 0 (the default): on the host."""
    flag = environ.get("C2V_DEVICE_TEXT", "0") or "0"
    if flag not in ("0", "1"):
        raise ValueError("C2V_DEVICE_TEXT must be 0 or 1, got %r" % flag)
    return flag == "1"


def word_prefixes(index_to_word, n_words: int, encoding: str, errors: str = "strict") -> Tuple[bytes, np.ndarray]:
    """The prefix of every word2vec row, `word + " "` encoded as the text file encodes it, concatenated, and their
    offsets [n_words + 1].  Asserts `i in index_to_word` for every row, as common.save_word2vec_file does."""
    parts = []
    for i in range(n_words):
        assert i in index_to_word
        parts.append((index_to_word[i] + " ").encode(encoding, errors))
    off = np.zeros(n_words + 1, dtype=np.int64)
    np.cumsum([len(p) for p in parts], out=off[1:])
    return b"".join(parts), off


class DeviceTextWriter:
    """Writes rows of device float32 matrices as text lines to `file` (a binary file object), formatted on `device`
    on the current stream.  close() writes what is still pending and frees the buffers; it does not close the file."""

    def __init__(self, file, device, chunk_bytes: int = CHUNK_BYTES):
        import torch
        self.torch = torch
        self.lib = load_library()
        self.file = file
        self.dev = torch.device(device)
        self.chunk_bytes = int(chunk_bytes)
        self._out = self._stage = self._ends = None
        self._pinned = [None, None]
        self._meta = [torch.zeros(2, dtype=torch.int64, pin_memory=True) for _ in range(2)]
        self._events = [torch.cuda.Event(), torch.cuda.Event()]
        self._slot = 0
        self._pending = None                       # (slot, rows) of the chunk whose text is not yet in the file
        self.peak_device_bytes = self.peak_host_bytes = 0
        self.bytes_written = 0

    # ---- buffers ----------------------------------------------------------------------------------------------------
    def device_bytes(self) -> int:
        """Device memory held now: the output text, the stage, the row ends (and the prefixes of a write_rows call)."""
        return int(sum(t.numel() * t.element_size() for t in (self._out, self._stage, self._ends) if t is not None))

    def host_bytes(self) -> int:
        """Page-locked host memory held now: the two text buffers and their read-backs."""
        return int(sum(t.numel() for t in self._pinned if t is not None) + 2 * 16)

    def _ensure(self, slot: int, rows: int, text_bytes: int, stage_bytes: int):
        torch = self.torch
        grow = lambda t, n, dt: t if t is not None and t.numel() >= n else torch.empty(n, dtype=dt, device=self.dev)
        self._out = grow(self._out, text_bytes, torch.uint8)
        self._stage = grow(self._stage, stage_bytes, torch.uint8)
        self._ends = grow(self._ends, rows + 1, torch.int64)
        p = self._pinned[slot]
        if p is None or p.numel() < text_bytes:    # never the pending chunk's slot
            self._pinned[slot] = None
            self._pinned[slot] = torch.empty(text_bytes, dtype=torch.uint8, pin_memory=True)
        self.peak_device_bytes = max(self.peak_device_bytes, self.device_bytes())
        self.peak_host_bytes = max(self.peak_host_bytes, self.host_bytes())

    # ---- writing ----------------------------------------------------------------------------------------------------
    def write_rows(self, x, prefixes: Optional[Tuple[bytes, np.ndarray]] = None):
        """Queues the lines of x [n, D] (float32, on the writer's device): each row's values joined by single spaces,
        then '\\n'; with prefixes = (blob, offsets [n + 1]) (word_prefixes), row r starts with blob[off[r], off[r + 1]).
        x may be freed once this returns: the work is ordered on the current stream."""
        torch = self.torch
        if x.dim() != 2 or x.dtype != torch.float32 or x.device != self.dev:
            raise ValueError("write_rows needs a 2-d float32 tensor on %s, got %s %s on %s" % (
                self.dev, tuple(x.shape), x.dtype, x.device))
        if x.shape[1] == 0:
            raise ValueError("write_rows needs at least one column")
        if x.stride(1) != 1:
            x = x.contiguous()
        n, D = int(x.shape[0]), int(x.shape[1])
        if n == 0:
            return
        per_row = D * VALUE_BYTES
        if prefixes is None:
            p_blob = p_off = None
            ends = np.arange(n + 1, dtype=np.int64) * per_row
        else:
            blob, off = prefixes
            off = np.ascontiguousarray(off, dtype=np.int64)
            if off.shape != (n + 1,) or off[0] != 0 or off[-1] != len(blob):
                raise ValueError("prefix offsets must be [n + 1], from 0 to the blob's length")
            p_blob = torch.frombuffer(bytearray(blob) if blob else bytearray(1), dtype=torch.uint8).to(self.dev)
            p_off = torch.from_numpy(off).to(self.dev)
            ends = off + np.arange(n + 1, dtype=np.int64) * per_row
        stream = torch.cuda.current_stream(self.dev)
        r0 = 0
        while r0 < n:
            # the rows whose text bound fits the chunk, and at least one
            r1 = max(r0 + 1, int(np.searchsorted(ends, ends[r0] + self.chunk_bytes, side="right")) - 1)
            rows, bound = r1 - r0, int(ends[r1] - ends[r0])
            slot = self._slot
            self._slot ^= 1
            self._ensure(slot, rows, bound, rows * per_row)
            rc = self.lib.c2v_text_format_rows(
                x[r0].data_ptr(), rows, D, x.stride(0), None if p_blob is None else p_blob.data_ptr(),
                None if p_off is None else p_off[r0].data_ptr(), self._stage.data_ptr(), self._stage.numel(),
                self._out.data_ptr(), bound, self._ends[1:].data_ptr(), self._ends.data_ptr(), stream.cuda_stream)
            if rc != 0:
                raise EngineError(rc, self.lib.c2v_last_error(None).decode())
            self._pinned[slot][:bound].copy_(self._out[:bound], non_blocking=True)
            self._meta[slot][0:1].copy_(self._ends[0:1], non_blocking=True)             # rows done
            self._meta[slot][1:2].copy_(self._ends[rows:rows + 1], non_blocking=True)   # the chunk's text bytes
            self._events[slot].record(stream)
            self._flush_pending()
            self._pending = (slot, rows)
            r0 = r1
        if p_blob is not None:
            # the prefixes are freed on return; what is queued on the stream is ordered before any reuse of that memory
            self.peak_device_bytes = max(self.peak_device_bytes, self.device_bytes() + p_blob.numel() + p_off.numel() * 8)

    def _flush_pending(self):
        if self._pending is None:
            return
        slot, rows = self._pending
        self._pending = None
        self._events[slot].synchronize()
        done, nbytes = (int(v) for v in self._meta[slot].tolist())
        if done != rows:
            raise RuntimeError("c2v_text_format_rows wrote %d of %d rows into a buffer sized for all of them" % (done, rows))
        self.file.write(memoryview(self._pinned[slot].numpy())[:nbytes])
        self.bytes_written += nbytes

    def close(self):
        """Writes the pending chunk and frees the buffers."""
        try:
            self._flush_pending()
        finally:
            self._out = self._stage = self._ends = None
            self._pinned = [None, None]

    def report(self) -> str:
        return "%.1f MB of text written; %.1f MB of device memory and %.1f MB of page-locked host memory held" % (
            self.bytes_written / 1e6, self.peak_device_bytes / 1e6, self.peak_host_bytes / 1e6)


def save_word2vec_file(output_file, index_to_word, table, chunk_bytes: int = CHUNK_BYTES) -> DeviceTextWriter:
    """common.save_word2vec_file with the rows of `table` (a device tensor [n_words, dim]) formatted on the GPU:
    output_file is the same text file, and it receives the same bytes.  Returns the writer, closed, for its report."""
    assert table.dim() == 2
    n_words, dim = (int(v) for v in table.shape)
    output_file.write("%d %d\n" % (n_words, dim))
    prefixes = word_prefixes(index_to_word, n_words, output_file.encoding, output_file.errors or "strict")
    output_file.flush()
    writer = DeviceTextWriter(output_file.buffer, table.device, chunk_bytes)
    try:
        writer.write_rows(table, prefixes)
    finally:
        writer.close()
    output_file.buffer.flush()
    return writer


def write_lines(file, x, chunk_bytes: int = CHUNK_BYTES, prefixes: Optional[Tuple[bytes, Sequence[int]]] = None):
    """The lines of one matrix written through a writer of its own (tests, tools)."""
    writer = DeviceTextWriter(file, x.device, chunk_bytes)
    try:
        writer.write_rows(x, prefixes)
    finally:
        writer.close()
    return writer
