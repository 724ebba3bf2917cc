"""`<corpus>.name_scores` and `<corpus>.nearest` written from device memory (DESIGN.md §6o).

With C2V_DEVICE_EVAL=1, `--score_names F.c2v` and `--nearest F.c2v` read F.c2v with the GPU evaluation reader and format
their lines on the GPU (c2v_name_scores_text, c2v_nearest_text; include/c2v_b200.h "Corpus text"): byte for byte what
name_scores.format_line and similarity.format_nearest_line write on the host.  LineStage brings each block of text back
through page-locked memory and writes it while the GPU works on the next one.  atomic_output gives both routes the host
route's outcome on a corpus that fails to read: no output file."""
from __future__ import annotations

import contextlib
import os

from .engine import EngineError, load_library

OUT_BYTES = 16 << 20          # the device text buffer a stage starts with; it grows to the largest block
NEAREST_ROWS = 1 << 16        # lines of `.nearest` formatted per call


@contextlib.contextmanager
def atomic_output(path: str):
    """A binary file that becomes `path` only when the block exits normally: the text goes to `path.<pid>.tmp` beside it,
    which is renamed over `path` at the end, or removed when the block raises (an earlier `path` is then left as it
    was)."""
    tmp = "%s.%d.tmp" % (path, os.getpid())
    f = open(tmp, "wb")
    try:
        yield f
        f.close()
        os.replace(tmp, path)
    except BaseException:
        f.close()
        with contextlib.suppress(OSError):
            os.unlink(tmp)
        raise


class LineStage:
    """Writes blocks of lines formatted on `device` to the binary file `file`.  emit(fmt) runs fmt(out, cap, total) --
    one c2v_*_text call into the device buffer out of cap bytes, its length to the page-locked int64 at total -- on the
    current stream, then writes the block the previous emit staged, then stages this one: the host writes block k while
    the GPU formats block k + 1.  close() writes the last block."""

    def __init__(self, file, device):
        import torch
        self.torch = torch
        self.lib = load_library()
        self.file = file
        self.dev = torch.device(device)
        self.out = None
        self.scratch = None
        self.pinned = [None, None]
        self.total = torch.zeros(1, dtype=torch.int64).pin_memory()
        self._slot = 0
        self._pending = None                       # memoryview of the staged block not yet written
        self.bytes_written = 0
        self.peak_device_bytes = self.peak_host_bytes = 0
        self.format_s = self.write_s = 0.0        # host time waiting for the format and copy, and in write()

    def _check(self, rc: int):
        if rc != 0:
            raise EngineError(rc, self.lib.c2v_last_error(None).decode())

    def scratch_for(self, rows: int):
        """Device scratch of at least c2v_corpus_text_scratch_bytes(rows) bytes: (pointer, bytes)."""
        n = int(self.lib.c2v_corpus_text_scratch_bytes(int(rows)))
        if self.scratch is None or self.scratch.numel() < n:
            self.scratch = None
            self.scratch = self.torch.empty(max(n, 1 << 16), dtype=self.torch.uint8, device=self.dev)
        return self.scratch.data_ptr(), int(self.scratch.numel())

    def _held(self):
        dev = sum(t.numel() for t in (self.out, self.scratch) if t is not None)
        host = sum(t.numel() for t in self.pinned if t is not None)
        self.peak_device_bytes = max(self.peak_device_bytes, dev)
        self.peak_host_bytes = max(self.peak_host_bytes, host)

    def emit(self, fmt):
        import time
        torch = self.torch
        if self.out is None:
            self.out = torch.empty(OUT_BYTES, dtype=torch.uint8, device=self.dev)
        stream = torch.cuda.current_stream(self.dev)
        fmt(self.out.data_ptr(), self.out.numel(), self.total.data_ptr())
        self._write_pending()
        t0 = time.perf_counter()
        stream.synchronize()
        total = int(self.total[0])
        if total > self.out.numel():               # the block did not fit: again into a buffer that holds it
            self.out = None
            self.out = torch.empty(total, dtype=torch.uint8, device=self.dev)
            fmt(self.out.data_ptr(), self.out.numel(), self.total.data_ptr())
            stream.synchronize()
        host = self.pinned[self._slot]
        if host is None or host.numel() < total:
            self.pinned[self._slot] = None
            host = self.pinned[self._slot] = torch.empty(max(total, 1 << 20), dtype=torch.uint8).pin_memory()
        host[:total].copy_(self.out[:total])
        self.format_s += time.perf_counter() - t0
        self._pending = memoryview(host.numpy())[:total]
        self._slot ^= 1
        self._held()

    def _write_pending(self):
        import time
        if self._pending is None:
            return
        t0 = time.perf_counter()
        self.file.write(self._pending)
        self.write_s += time.perf_counter() - t0
        self.bytes_written += len(self._pending)
        self._pending = None

    def close(self):
        """Writes the staged block and frees the buffers."""
        try:
            self._write_pending()
        finally:
            self.out = self.scratch = None
            self.pinned = [None, None]
