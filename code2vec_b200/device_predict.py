"""`--predict` on the GPU (DESIGN.md §6i): extractor output read into device memory, its methods predicted in batches of
TEST_BATCH_SIZE rows and their text formatted on the device (include/c2v_b200.h, "Device predict"), byte for byte what
__main__.print_predictions writes for the same input.

The input is held in host memory (the host route holds all its lines too) and goes to the device in chunks of at most
CHUNK_BYTES of whole lines (chunk_ranges), so the device memory does not grow with the input:
  pass 1 : every chunk is scanned (the source's newline rule, rstrip, fields, the three-part check) and its contexts'
           keys recorded in the key -> last path table that print_predictions' `unhash` dict is; then every chunk again
           hands the table the texts of the paths it names.  A malformed context raises ValueError here, before a byte
           is written.
  pass 2 : per chunk and per batch of its methods, c2v_pred_rows builds the model input rows, engine.forward /
           engine.topk (what c2v_predict_batch_host runs) predict them, and c2v_pred_format ranks each row's attention
           and writes its block.  Two page-locked buffers take the text: the host writes batch i while the GPU predicts
           and formats batch i + 1.

Inputs the kernels do not restate go through the host route whole, with a log line: a byte >= 0x80 (Unicode rstrip,
isdigit and decoding), and a path whose key the int32-keyed table cannot hold (a numeric path that is not the canonical
decimal of an int32, such as "007", whose key is its own text, or a path of 1 MB or more).  Code2VecModel uses this route when C2V_DEVICE_PREDICT=1."""
from __future__ import annotations

import ctypes as C
import io

import numpy as np

from .engine import EngineError, load_library

SHOW_TOP_CONTEXTS = 10            # __main__.SHOW_TOP_CONTEXTS
OUT_BYTES = 64 << 20              # the device text buffer of a batch to start with (grown when a batch needs more)
CHUNK_BYTES = 64 << 20            # the most input the device holds at once (a longer line makes its chunk longer)

KIND_METHOD, KIND_MALFORMED, KIND_ODD_KEY = 1, 2, 3          # c2v_pred_line_info's kinds (0: a skipped line)
SCAN, KEYS, PATHS = 0, 1, 2                                    # C2V_PRED_SCAN, C2V_PRED_KEYS, C2V_PRED_PATHS


def chunk_ranges(data: bytes, chunk_bytes: int):
    """[lo, hi) byte ranges that cut `data` into chunks of whole lines: each ends just after a '\n' (which ends a line
    under both newline rules and never splits a "\r\n") or at the end of the data, and is at most chunk_bytes long
    unless one line is longer."""
    out, lo, n = [], 0, len(data)
    while lo < n:
        hi = min(lo + chunk_bytes, n)
        if hi < n:
            cut = data.rfind(b"\n", lo, hi)
            if cut < 0:
                cut = data.find(b"\n", hi)
            hi = n if cut < 0 else cut + 1
        out.append((lo, hi))
        lo = hi
    return out


def device_predict_flag(environ) -> bool:
    """C2V_DEVICE_PREDICT=1: `--predict` reads, predicts and formats on the GPU; 0 (the default): on the host."""
    flag = environ.get("C2V_DEVICE_PREDICT", "0") or "0"
    if flag not in ("0", "1"):
        raise ValueError("C2V_DEVICE_PREDICT must be 0 or 1, got %r" % flag)
    return flag == "1"


def split_source_lines(data: bytes, universal_newlines: bool):
    """The lines Python iterates over for `data`: a file opened with open(path, "r") (universal newlines: "\\n", "\\r\\n"
    and a lone "\\r" end a line and read as "\\n"), or sys.stdin, whose lines end at "\\n" only."""
    text = data.decode("utf-8")
    return io.StringIO(text, newline=None if universal_newlines else "\n")


def target_reprs(target_vocab):
    """(bytes, offsets) of str(word.split("|")) for every target word: the `%s` of a "predicted:" line."""
    enc = [str(target_vocab.index_to_word[i].split("|")).encode("utf-8") for i in range(target_vocab.size)]
    off = np.zeros(len(enc) + 1, dtype=np.int64)
    np.cumsum([len(b) for b in enc], out=off[1:])
    return np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8), off


class DevicePredictor:
    """The device route of one model: made once per model, freed by close() (Code2VecModel.close_session)."""

    def __init__(self, model, normalize: int):
        import torch
        from .path_context_reader import EstimatorAction, PathContextReader
        from .b200_model import _EvaluateInputFormer
        self.torch = torch
        self.model = model
        self.engine = model.engine
        self.dev = self.engine.dev
        self.normalize = int(normalize)
        cfg = model.config
        self.C = cfg.MAX_CONTEXTS
        self.B = max(1, cfg.TEST_BATCH_SIZE)
        self.lib = load_library()
        # any reader of the model with the native tensoriser: its vocabulary tables are what the device looks words up in
        reader = PathContextReader(vocabs=model.vocabs, model_input_tensors_former=_EvaluateInputFormer(), config=cfg,
                                   estimator_action=EstimatorAction.Evaluate)
        self.vocabs = model._shared_device_vocabs(reader)
        self.h = C.c_void_p()
        self._check(self.lib.c2v_pred_create(self.engine.device, self.C, C.byref(self.vocabs.structs[0]),
                                             C.byref(self.vocabs.structs[1]), C.byref(self.h)))
        tv = model.vocabs.target_vocab
        repr_bytes, repr_off = target_reprs(tv)
        self.oov = int(tv.word_to_index[tv.special_words.OOV])
        self._check(self.lib.c2v_pred_set_targets(self.h, tv.size, repr_bytes.ctypes.data, repr_off.ctypes.data, self.oov,
                                                  None))
        self.k = min(self.engine.dims.top_k, self.engine.dims.target_vocab)
        B, Cn = self.B, self.C
        with torch.cuda.device(self.dev):
            self.rows = [torch.empty((B, Cn), dtype=torch.int32, device=self.dev) for _ in range(3)]
            self.mask = torch.empty((B, Cn), dtype=torch.float32, device=self.dev)
        self.out_dev = None                     # device text of one batch, grown as needed
        self.out_host = [None, None]            # the two page-locked buffers
        self.scalars = torch.zeros(2, dtype=torch.int64).pin_memory()      # (text length, bad row) of a batch
        self.pinned_bytes = 0
        self.ran = []                           # per run(): True on the device, False when handed to the host route

    def _check(self, rc):
        if rc != 0:
            raise EngineError(rc, self.lib.c2v_last_error(None).decode())

    def device_bytes(self) -> int:
        own = int(self.lib.c2v_pred_device_bytes(self.h)) if self.h else 0
        return own + (self.out_dev.numel() if self.out_dev is not None else 0) + \
            sum(t.numel() * 4 for t in self.rows) + self.mask.numel() * 4

    def close(self):
        if self.h:
            self.lib.c2v_pred_destroy(self.h)
            self.h = C.c_void_p()
        self.out_dev = None
        self.out_host = [None, None]

    # ---- chunks --------------------------------------------------------------------------------------------------
    def _chunk(self, data: bytes, lo: int, hi: int, universal_newlines: bool, mode: int) -> int:
        """c2v_pred_chunk on data[lo:hi]; the chunk's number of lines."""
        buf = np.frombuffer(data, dtype=np.uint8, count=hi - lo, offset=lo) if hi > lo else np.zeros(1, dtype=np.uint8)
        n_lines = C.c_int64()
        self._check(self.lib.c2v_pred_chunk(self.h, buf.ctypes.data, hi - lo, lo, int(universal_newlines), mode,
                                            C.byref(n_lines), self.engine._stream()))
        return int(n_lines.value)

    def _line_info(self, n_lines: int):
        lo, hi = np.zeros(n_lines, dtype=np.int64), np.zeros(n_lines, dtype=np.int64)
        kind, kept = np.zeros(n_lines, dtype=np.int32), np.zeros(n_lines, dtype=np.int32)
        if n_lines:
            self._check(self.lib.c2v_pred_line_info(self.h, lo.ctypes.data, hi.ctypes.data, kind.ctypes.data,
                                                    kept.ctypes.data))
        return lo, hi, kind, kept

    def _host_buffer(self, i: int, nbytes: int):
        cur = self.out_host[i]
        if cur is None or cur.numel() < nbytes:
            self.out_host[i] = self.torch.empty(max(nbytes, 1 << 20), dtype=self.torch.uint8).pin_memory()
            self.pinned_bytes = sum(b.numel() for b in self.out_host if b is not None)
        return self.out_host[i]

    # ---- both passes -------------------------------------------------------------------------------------------------
    def run(self, data: bytes, universal_newlines: bool, out, want_code: bool, chunk_bytes: int = None) -> bool:
        """Writes the text of every method of `data` to the binary stream `out`.  False (nothing written) when the input
        needs the host route; ValueError (nothing written) for a malformed context."""
        ok = self._run(data, universal_newlines, out, want_code, CHUNK_BYTES if chunk_bytes is None else chunk_bytes)
        self.ran.append(ok)
        return ok

    def _run(self, data, universal_newlines, out, want_code, chunk_bytes) -> bool:
        torch = self.torch
        if np.frombuffer(data, dtype=np.uint8).max(initial=0) >= 0x80:
            return False
        chunks = chunk_ranges(data, chunk_bytes)
        # pass 1: every line's kind and every key's last path
        self._check(self.lib.c2v_pred_reset_keys(self.h, self.engine._stream()))
        methods, line0 = [], 0
        for lo, hi in chunks:
            n_lines = self._chunk(data, lo, hi, universal_newlines, KEYS)
            l_lo, l_hi, kind, _ = self._line_info(n_lines)
            if (kind == KIND_ODD_KEY).any():
                return False
            bad = np.flatnonzero(kind == KIND_MALFORMED)
            if bad.size:
                j = int(bad[0])
                raise ValueError("line %d of the predict input has a context without exactly three comma-separated parts: "
                                 "%r" % (line0 + j + 1, data[lo + l_lo[j]:lo + l_hi[j]].decode("ascii")))
            methods.append((line0, np.flatnonzero(kind == KIND_METHOD).astype(np.int64)))
            line0 += n_lines
        self._check(self.lib.c2v_pred_seal_keys(self.h, self.engine._stream()))
        for lo, hi in chunks:
            self._chunk(data, lo, hi, universal_newlines, PATHS)
        # pass 2: per chunk, its methods in batches
        e = self.engine
        e.set_option("math_mode", self.model._math_eval)
        stream = torch.cuda.current_stream(self.dev)
        if self.out_dev is None:
            self.out_dev = torch.empty(OUT_BYTES, dtype=torch.uint8, device=self.dev)
        written = None                          # the text of the batch the host writes next
        b = 0
        for (lo, hi), (first_line, rows) in zip(chunks, methods):
            if rows.size == 0:
                continue
            self._chunk(data, lo, hi, universal_newlines, SCAN)
            for s in range(0, rows.size, self.B):
                n = min(self.B, rows.size - s)
                lines = np.ascontiguousarray(rows[s:s + n])
                src, pth, tgt = (t[:n] for t in self.rows)
                mask = self.mask[:n]
                self._check(self.lib.c2v_pred_rows(self.h, lines.ctypes.data, n, src.data_ptr(), pth.data_ptr(),
                                                   tgt.data_ptr(), mask.data_ptr(), e._stream()))
                code, attn = e.forward(src, pth, tgt, mask, want_attention=True)
                idx, val = e.topk(code, normalize=self.normalize)

                def fmt():
                    self._check(self.lib.c2v_pred_format(
                        self.h, n, idx.data_ptr(), val.data_ptr(), self.k, attn.data_ptr(),
                        code.data_ptr() if want_code else None, e.dims.code_dim, self.out_dev.data_ptr(),
                        self.out_dev.numel(), self.scalars.data_ptr(), self.scalars.data_ptr() + 8, e._stream()))
                fmt()
                if written is not None:         # the previous batch goes out while the GPU formats this one
                    out.write(written)
                    written = None
                stream.synchronize()
                total, bad_row = int(self.scalars[0]), int(self.scalars[1])
                if bad_row < n:
                    raise RuntimeError("the attention of the method on line %d of the predict input is NaN for some "
                                       "contexts only: the engine's forward pass is at fault"
                                       % (first_line + int(lines[bad_row]) + 1))
                if total > self.out_dev.numel():    # the text did not fit: again into a buffer that holds it
                    self.out_dev = None
                    self.out_dev = torch.empty(total, dtype=torch.uint8, device=self.dev)
                    fmt()
                    stream.synchronize()
                host = self._host_buffer(b % 2, total)
                host[:total].copy_(self.out_dev[:total])
                written = memoryview(host.numpy())[:total]
                b += 1
        if written is not None:
            out.write(written)
        return True
