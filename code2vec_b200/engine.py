"""ctypes binding of libc2v_b200.so (include/c2v_b200.h) and the storage that goes with it.

PyTorch is used for device/pinned memory, streams and (elsewhere) torch.distributed only; every
arithmetic step of the hot path runs inside the C-ABI library's CUDA kernels.  There is no CPU
fallback: if the library cannot be loaded this module raises.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np

from . import build as _build

PARAM_NAMES = ("tok", "path", "tgt", "W", "a")

MATH_FP32 = 0
MATH_TF32 = 1
MATH_3XTF32 = 2
MATH_MODES = {"fp32": MATH_FP32, "tf32": MATH_TF32, "3xtf32": MATH_3XTF32}


class c2v_dims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("token_vocab", "path_vocab", "target_vocab", "embed_dim",
                                         "code_dim", "max_contexts", "max_batch", "top_k")]


class c2v_tensors(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in PARAM_NAMES]


class c2v_table_shards(C.Structure):
    _fields_ = [("world", C.c_int32), ("rank", C.c_int32), ("tok", C.c_void_p * 8), ("path", C.c_void_p * 8)]


class c2v_reader_vocab(C.Structure):
    _fields_ = [("slots", C.c_void_p), ("bytes", C.c_void_p), ("mask", C.c_uint64), ("oov", C.c_int32), ("pad", C.c_int32)]


class c2v_reader_share_status(C.Structure):
    _fields_ = [("rows", C.c_int64), ("records", C.c_int64), ("kept", C.c_int64), ("newlines", C.c_int64),
                ("bad_line", C.c_int64), ("bad_kind", C.c_int32), ("overflow", C.c_int32)]


class c2v_prep_status(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("lines", "bad_utf8", "bad_line", "long_lines", "seen", "kept", "written", "empty",
                                         "longest", "keys", "slots", "rehashes")]


class _DeviceArray:
    """A raw device allocation presented through __cuda_array_interface__ so torch can view it."""

    def __init__(self, ptr: int, shape):
        self.__cuda_array_interface__ = {"shape": tuple(int(x) for x in shape), "typestr": "<f4", "data": (int(ptr), False),
                                         "version": 2, "strides": None}


# every symbol include/c2v_b200.h declares: (restype, argtypes)
_P = C.c_void_p
_I32 = C.c_int32
_SIGNATURES = {
    "c2v_abi_version": (C.c_int, []),
    "c2v_last_error": (C.c_char_p, [_P]),
    "c2v_workspace_bytes": (C.c_size_t, [C.POINTER(c2v_dims)]),
    "c2v_create": (C.c_int, [C.POINTER(c2v_dims), C.c_int, C.POINTER(_P)]),
    "c2v_destroy": (None, [_P]),
    "c2v_bind_workspace": (C.c_int, [_P, _P, C.c_size_t]),
    "c2v_bind_params": (C.c_int, [_P, C.POINTER(c2v_tensors)]),
    "c2v_bind_grads": (C.c_int, [_P, C.POINTER(c2v_tensors)]),
    "c2v_bind_adam_state": (C.c_int, [_P, C.POINTER(c2v_tensors), C.POINTER(c2v_tensors)]),
    "c2v_set_option": (C.c_int, [_P, C.c_char_p, C.c_int64]),
    "c2v_get_option": (C.c_int, [_P, C.c_char_p, C.POINTER(C.c_int64)]),
    "c2v_forward": (C.c_int, [_P, _P, _P, _P, _P, _I32, _P, _P, _P]),
    "c2v_topk": (C.c_int, [_P, _P, _I32, _P, _P, _I32, _P]),
    "c2v_loss": (C.c_int, [_P, _P, _P, _I32, _P, _P]),
    "c2v_name_scores": (C.c_int, [_P, _P, _P, _I32, _P, _P, _P, _P, _P]),
    "c2v_train_step": (C.c_int, [_P, _P, _P, _P, _P, _P, _I32, C.c_float, C.c_uint64, C.c_uint64, _P, _P, _P]),
    "c2v_sampled_train_step": (C.c_int, [_P, _P, _P, _P, _P, _P, _I32, _P, _I32, _P, _P, C.c_float,
                                         C.c_uint64, C.c_uint64, _P, _P, _P]),
    "c2v_sample_log_uniform": (C.c_int, [_P, _I32, _P, _I32, C.c_uint64, C.c_uint64, _P, _P, _P, _P, _P]),
    "c2v_sample_log_uniform_vocab": (C.c_int, [_P, _I32, _I32, _P, _I32, C.c_uint64, C.c_uint64, _P, _P, _P, _P, _P]),
    "c2v_adam_step": (C.c_int, [_P, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int64, _P]),
    "c2v_arm_target_adam": (C.c_int, [_P, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int64]),
    "c2v_hint_next_batch": (C.c_int, [_P, _P, _P, _P, _I32]),
    "c2v_hint_next_batch_host": (C.c_int, [_P, _P, _P, _P, _I32, _P]),
    "c2v_adam_step_range": (C.c_int, [_P, _P, _P, _P, _P, C.c_size_t, C.c_float, C.c_float, C.c_float, C.c_float,
                                      C.c_int64, _I32, _P]),
    "c2v_bind_table_shards": (C.c_int, [_P, C.POINTER(c2v_table_shards), C.POINTER(c2v_table_shards), C.c_float]),
    "c2v_scatter_inbox_bytes": (C.c_size_t, [C.POINTER(c2v_dims), _I32]),
    "c2v_bind_scatter_inbox": (C.c_int, [_P, C.POINTER(_P), _I32, _I32]),
    "c2v_apply_scatter_inbox": (C.c_int, [_P, _P]),
    "c2v_ipc_alloc": (C.c_int, [C.c_int, C.c_size_t, C.POINTER(_P), C.c_char_p]),
    "c2v_ipc_open": (C.c_int, [C.c_int, C.c_char_p, C.POINTER(_P)]),
    "c2v_ipc_close": (C.c_int, [C.c_int, _P]),
    "c2v_ipc_free": (C.c_int, [C.c_int, _P]),
    "c2v_train_batch_host": (C.c_int, [_P, _P, _P, _P, _P, _P, _I32, C.c_float, C.c_uint64, C.c_int64,
                                       C.c_float, C.c_float, C.c_float, C.c_float, _P, _P]),
    "c2v_train_batch_async": (C.c_int, [_P, _P, _P, _P, _P, _P, _I32, C.c_float, C.c_uint64, C.c_int64,
                                        C.c_float, C.c_float, C.c_float, C.c_float, _P, _P, _P]),
    "c2v_predict_batch_host": (C.c_int, [_P, _P, _P, _P, _P, _I32, _I32, _P, _P, _P, _P, _P]),
    "c2v_selftest_gemm": (C.c_int, [_P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P, C.c_size_t, _P, C.c_size_t,
                                    _P, C.c_size_t, _P]),
    "c2v_selftest_gemm3": (C.c_int, [_P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P, _P, C.c_size_t, _P, _P, C.c_size_t,
                                     _P, C.c_size_t, _P]),
    "c2v_selftest_gemm_bt": (C.c_int, [_P, _I32, _I32, _I32, _P, C.c_size_t, _P, C.c_size_t, _P, C.c_size_t, _P, C.c_size_t,
                                       _P]),
    "c2v_selftest_split": (C.c_int, [_P, _P, _P, _P, C.c_size_t, _P]),
    "c2v_selftest_transpose": (C.c_int, [_P, _P, _I32, _I32, _P, _P, C.c_size_t, _P]),
    "c2v_selftest_target_t": (C.c_int, [_P, _I32, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "c2v_selftest_row_sum": (C.c_int, [_P, _I32, _P, _P, _I32, _P, _P]),
    "c2v_selftest_exchange_push": (C.c_int, [_P, _P, _P, _I32, _P, _P, _I32, _P]),
    "c2v_set_event": (C.c_int, [_P, C.c_char_p, _P]),
    "c2v_sync_tables": (C.c_int, [_P, _P]),
    "c2v_context_forward": (C.c_int, [_P, _P, _P, _P, _P, _I32, C.c_float, C.c_uint64, C.c_uint64, _P, _P, _P]),
    "c2v_target_forward": (C.c_int, [_P, _P, _I32, _P, _I32, _P, _P, _P, _P]),
    "c2v_lse_combine": (C.c_int, [_P, _P, _P, _I32, _I32, _P, C.c_float, _P, _P, _P]),
    "c2v_target_backward": (C.c_int, [_P, _P, _I32, _P, _P, _I32, C.c_float, _P, _P]),
    "c2v_context_backward": (C.c_int, [_P, _P, _P, _P, _P, _I32, C.c_float, C.c_uint64, C.c_uint64, _P, _P, _P]),
    "c2v_sampled_pack_rows": (C.c_int, [_P, _P, _I32, _P, _I32, _I32, _P, _P, _P]),
    "c2v_sampled_target_step": (C.c_int, [_P, _P, _I32, _P, _P, _I32, _P, _P, _P, _P, C.c_float, _P, _P, _P, _P, _P]),
    "c2v_sampled_target_fold": (C.c_int, [_P, _P, _P, _I32, _P, _I32, _P, _I32, _I32, _P, _P, _P]),
    "c2v_topk_partial": (C.c_int, [_P, _P, _I32, _I32, _I32, _P, _P, _P, _P, _P]),
    "c2v_topk_merge": (C.c_int, [_P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P, _P, _P]),
    "c2v_launch_count": (C.c_int64, [_P]),
    "c2v_phase_count": (C.c_int, []),
    "c2v_phase_name": (C.c_char_p, [C.c_int]),
    "c2v_phase_stats": (C.c_int, [_P, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int64), C.c_int]),
    # device reader (device_reader.py)
    "c2v_reader_create": (C.c_int, [_I32, C.POINTER(c2v_reader_vocab), C.POINTER(c2v_reader_vocab),
                                    C.POINTER(c2v_reader_vocab), C.c_int, C.POINTER(_P)]),
    "c2v_reader_destroy": (None, [_P]),
    "c2v_reader_parse_chunk": (C.c_int, [_P, _P, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(_I32), _P]),
    "c2v_reader_draw": (C.c_int, [_P, _P, _I32, _I32, _I32, _P, _P, _P, _P, _P, _P]),
    "c2v_reader_live_rows": (C.c_int64, [_P]),
    "c2v_reader_device_bytes": (C.c_size_t, [_P]),
    "c2v_reader_stage_bytes": (C.c_size_t, [_I32, C.c_int64]),
    "c2v_reader_parse_share": (C.c_int, [_P, _P, C.c_int64, C.c_int64, _P, C.c_int64, C.POINTER(c2v_reader_share_status),
                                         _P]),
    "c2v_reader_commit_shares": (C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_int64), _I32, C.POINTER(C.c_int64), _P]),
    "c2v_reader_eval_tables": (C.c_int, [_P, _I32, _P, _P, _P, _P, _P, _P]),
    "c2v_reader_eval_append": (C.c_int, [_P, _P, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                         C.POINTER(C.c_int64), C.POINTER(_I32), _P]),
    "c2v_reader_eval_take": (C.c_int, [_P, _I32, _P, _P, _P, _P, _P, _P, _P, C.c_int64, _P]),
    "c2v_reader_eval_queued": (C.c_int64, [_P]),
    "c2v_reader_eval_score": (C.c_int, [_P, _P, _I32, _I32, _P, _P, _P, _P, _P, _P, _P]),
    "c2v_reader_eval_check_utf8": (C.c_int, [_P, C.c_int64, _P, C.c_int64, C.POINTER(C.c_int64), _P]),
    "c2v_reader_eval_words": (C.c_int, [_P, C.POINTER(_P), C.POINTER(_P), C.POINTER(_I32)]),
    # text of float32 matrices (text_export.py)
    "c2v_text_format_rows": (C.c_int, [_P, C.c_int64, _I32, C.c_int64, _P, _P, _P, C.c_size_t, _P, C.c_int64, _P, _P,
                                       _P]),
    "c2v_selftest_format_floats": (C.c_int, [_P, C.c_int64, _P, _P]),
    # CRC-32C of tensor bundle entries (tf_bundle.py)
    "c2v_crc32c_rows": (C.c_int, [_P, C.c_int64, C.c_int64, C.c_int64, _P, _P]),
    "c2v_crc32c_combine": (C.c_int, [_P, C.c_int64, C.c_int64, _P, _P]),
    # the Keras output kernel's transpose (keras_ckpt.py)
    "c2v_rows_to_cols": (C.c_int, [_P, C.c_int64, C.c_int64, _P, C.c_int64, C.c_int64, _P]),
    "c2v_cols_to_rows": (C.c_int, [_P, C.c_int64, C.c_int64, C.c_int64, C.c_int64, _P, _P]),
    # preprocessing (device_preprocess.py)
    "c2v_prep_create": (C.c_int, [C.c_int, C.POINTER(_P)]),
    "c2v_prep_destroy": (None, [_P]),
    "c2v_prep_device_bytes": (C.c_size_t, [_P]),
    "c2v_prep_count_chunk": (C.c_int, [_P, _P, C.c_int64, C.c_int64, C.POINTER(c2v_prep_status), _P]),
    "c2v_prep_histogram": (C.c_int, [_P, _I32, C.POINTER(_P), C.POINTER(C.c_int64), _P]),
    "c2v_prep_classify_chunk": (C.c_int, [_P, _P, C.c_int64, _I32, C.POINTER(c2v_reader_vocab), C.POINTER(c2v_reader_vocab),
                                          C.POINTER(c2v_prep_status), _P]),
    "c2v_prep_long_lines": (C.c_int, [_P, _P, _P, _P, _P]),
    "c2v_prep_assemble": (C.c_int, [_P, _P, _P, C.POINTER(_P), C.POINTER(C.c_int64), _P]),
    # nearest neighbours (similarity.py)
    "c2v_knn_create": (C.c_int, [C.c_int, C.POINTER(_P)]),
    "c2v_knn_destroy": (None, [_P]),
    "c2v_knn_device_bytes": (C.c_size_t, [_P]),
    "c2v_knn_bind_table": (C.c_int, [_P, _P, C.c_int64, _I32, C.c_int64, _I32, _P]),
    "c2v_knn_queries": (C.c_int, [_P, _P, _P, _P, _I32, _P, _P]),
    "c2v_knn_search": (C.c_int, [_P, _P, _I32, C.c_int64, _I32, _P, _P, _I32, _P, _P, _P]),
    "c2v_knn_profile": (C.c_int, [_P, _I32, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    # device predict (device_predict.py)
    "c2v_pred_create": (C.c_int, [C.c_int, _I32, C.POINTER(c2v_reader_vocab), C.POINTER(c2v_reader_vocab), C.POINTER(_P)]),
    "c2v_pred_destroy": (None, [_P]),
    "c2v_pred_device_bytes": (C.c_size_t, [_P]),
    "c2v_pred_set_targets": (C.c_int, [_P, _I32, _P, _P, _I32, _P]),
    "c2v_pred_reset_keys": (C.c_int, [_P, _P]),
    "c2v_pred_chunk": (C.c_int, [_P, _P, C.c_int64, C.c_int64, _I32, _I32, C.POINTER(C.c_int64), _P]),
    "c2v_pred_seal_keys": (C.c_int, [_P, _P]),
    "c2v_pred_line_info": (C.c_int, [_P, _P, _P, _P, _P]),
    "c2v_pred_rows": (C.c_int, [_P, _P, _I32, _P, _P, _P, _P, _P]),
    "c2v_pred_format": (C.c_int, [_P, _I32, _P, _P, _I32, _P, _P, _I32, _P, C.c_int64, _P, _P, _P]),
    "c2v_selftest_format_fixed": (C.c_int, [_P, C.c_int64, _P, _P]),
    # corpus text (corpus_text.py)
    "c2v_corpus_text_scratch_bytes": (C.c_size_t, [C.c_int64]),
    "c2v_name_scores_text": (C.c_int, [_I32, _P, _P, _P, _I32, _P, _P, _P, _P, _P, _P, _I32, _P, C.c_size_t, _P,
                                       C.c_int64, _P, _P]),
    "c2v_nearest_text": (C.c_int, [C.c_int64, C.c_int64, C.c_int64, _I32, _P, _P, _P, _P, _P, C.c_size_t, _P, C.c_int64,
                                   _P, _P]),
}

_lib = None


def library_path() -> str:
    return _build.LIB_PATH


def load_library():
    """Loads (building first if the in-tree .so is missing or stale) and types the C ABI."""
    global _lib
    if _lib is not None:
        return _lib
    if _build.needs_build():
        _build.build()
    if not os.path.exists(_build.LIB_PATH):
        raise RuntimeError("libc2v_b200.so is missing; run `python -m code2vec_b200.build`")
    lib = C.CDLL(_build.LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the header and the library disagree
        fn.restype = res
        fn.argtypes = args
    if lib.c2v_abi_version() != 1:
        raise RuntimeError("libc2v_b200.so ABI version mismatch")
    _lib = lib
    return lib


class EngineError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__("c2v error %d: %s" % (code, msg))
        self.code = code


@dataclass
class EngineDims:
    token_vocab: int
    path_vocab: int
    target_vocab: int
    embed_dim: int
    code_dim: int
    max_contexts: int
    max_batch: int
    top_k: int = 10

    def shapes(self) -> Dict[str, Tuple[int, ...]]:
        d, D = self.embed_dim, self.code_dim
        return {"tok": (self.token_vocab, d), "path": (self.path_vocab, d), "tgt": (self.target_vocab, D),
                "W": (3 * d, D), "a": (D,)}

    def to_c(self) -> c2v_dims:
        return c2v_dims(self.token_vocab, self.path_vocab, self.target_vocab, self.embed_dim, self.code_dim,
                        self.max_contexts, self.max_batch, self.top_k)


def _ptr(t) -> Optional[int]:
    return None if t is None else t.data_ptr()


class PathAttentionEngine:
    """Owns the storage (torch tensors) and one c2v_engine handle on one GPU."""

    def __init__(self, dims: EngineDims, device: int = 0, training: bool = True):
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError("PathAttentionEngine needs a CUDA device (H100); no CPU fallback exists")
        self.torch = torch
        self.lib = load_library()
        self.dims = dims
        self.device = int(device)
        self.dev = torch.device("cuda", self.device)
        self.training = training
        cd = dims.to_c()
        h = _P()
        rc = self.lib.c2v_create(C.byref(cd), self.device, C.byref(h))
        if rc != 0:
            raise EngineError(rc, self.lib.c2v_last_error(None).decode())
        self.h = h
        f32 = torch.float32
        with torch.cuda.device(self.dev):
            wbytes = self.lib.c2v_workspace_bytes(C.byref(cd))
            self.workspace = torch.empty(wbytes, dtype=torch.uint8, device=self.dev)
            self._check(self.lib.c2v_bind_workspace(self.h, self.workspace.data_ptr(), wbytes))
            # One flat fp32 buffer per role (parameters, gradients, Adam m, Adam v) with the five
            # tensors as views at 256-byte-aligned offsets: a data-parallel run can then
            # reduce-scatter / all-gather the whole model in one collective and run Adam on a slice.
            self.flat_params, self.params = self._alloc_flat()
            self._check(self.lib.c2v_bind_params(self.h, C.byref(self._tensors(self.params))))
            self.grads = self.adam_m = self.adam_v = None
            self.flat_grads = self.flat_m = self.flat_v = None
            if training:
                self.flat_grads, self.grads = self._alloc_flat()
                self.flat_m, self.adam_m = self._alloc_flat()
                self.flat_v, self.adam_v = self._alloc_flat()
                self._check(self.lib.c2v_bind_grads(self.h, C.byref(self._tensors(self.grads))))
                self._check(self.lib.c2v_bind_adam_state(self.h, C.byref(self._tensors(self.adam_m)),
                                                         C.byref(self._tensors(self.adam_v))))
            self._loss = torch.zeros(1, dtype=f32, device=self.dev)
        self.adam_t = 0

    # ---- plumbing -------------------------------------------------------------------------
    FLAT_ALIGN = 1024          # floats: keeps every view 256-byte aligned and any world size <= 256 dividing the total

    FLAT_ORDER = ("tgt", "tok", "path", "W", "a")   # target table first: its gradient is complete first (bucket A)

    def flat_layout(self):
        """[(name, offset, numel)] of the five tensors inside a flat buffer, and its padded length."""
        out, off = [], 0
        shapes = self.dims.shapes()
        for k in self.FLAT_ORDER:
            n = int(np.prod(shapes[k]))
            out.append((k, off, n))
            off = (off + n + self.FLAT_ALIGN - 1) // self.FLAT_ALIGN * self.FLAT_ALIGN
        return out, off

    def bucket_bounds(self):
        """Two gradient buckets of the flat buffer: A = target table (ready right after the dY GEMM),
        B = token/path tables, TRANSFORM, ATTENTION (ready at the end of the backward pass)."""
        layout, total = self.flat_layout()
        split = layout[1][1]            # offset of the first tensor after `tgt`
        return (0, split), (split, total)

    def set_event(self, name: str, event) -> None:
        """Ask the engine to record `event` (torch.cuda.Event) on the launching stream at a named point
        of c2v_train_step ("target_grads_ready": right after dY is complete)."""
        event.record(self.torch.cuda.current_stream(self.dev))          # forces creation of the cudaEvent_t
        self._events = getattr(self, "_events", {})
        self._events[name] = event
        self._check(self.lib.c2v_set_event(self.h, name.encode(), event.cuda_event))

    def _alloc_flat(self):
        torch = self.torch
        layout, total = self.flat_layout()
        flat = torch.zeros(total, dtype=torch.float32, device=self.dev)
        shp = self.dims.shapes()
        views = {k: flat[off:off + n].view(shp[k]) for k, off, n in layout}
        return flat, views

    @staticmethod
    def _tensors(d) -> c2v_tensors:
        return c2v_tensors(*[d[k].data_ptr() for k in PARAM_NAMES])

    def _check(self, rc: int):
        if rc != 0:
            raise EngineError(rc, self.lib.c2v_last_error(self.h).decode())

    def _stream(self) -> int:
        return self.torch.cuda.current_stream(self.dev).cuda_stream

    def close(self):
        if getattr(self, "h", None):
            self.lib.c2v_destroy(self.h)
            self.h = None
            # peers' shards first (unmap), then this rank's own allocations
            for p in getattr(self, "_ipc_opened", []):
                self.lib.c2v_ipc_close(self.device, p)
            self._ipc_opened = []
            self.shard_params = self.shard_grads = None          # views of the allocations freed below
            for p in getattr(self, "_ipc_owned", []):
                self.lib.c2v_ipc_free(self.device, p)
            self._ipc_owned = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_option(self, key: str, value: int):
        self._check(self.lib.c2v_set_option(self.h, key.encode(), int(value)))

    def get_option(self, key: str) -> int:
        v = C.c_int64()
        self._check(self.lib.c2v_get_option(self.h, key.encode(), C.byref(v)))
        return v.value

    @property
    def launch_count(self) -> int:
        return int(self.lib.c2v_launch_count(self.h))

    def selftest_split(self, x):
        """Test hook: the 3xTF32 operand split of a device tensor -> (hi, lo)."""
        hi, lo = self.torch.empty_like(x), self.torch.empty_like(x)
        self._check(self.lib.c2v_selftest_split(self.h, x.data_ptr(), hi.data_ptr(), lo.data_ptr(), x.numel(), self._stream()))
        return hi, lo

    def selftest_transpose(self, x, ld_t: int, split: bool = False):
        """Test hook: the K-major copy [cols, ld_t] the engine makes of a row-major [rows, cols] operand (c2v_selftest_transpose);
        with split, the transposed 3xTF32 split -> (hi, lo).  Columns rows .. ld_t-1 are left as torch.empty made them."""
        rows, cols = x.shape
        out = [self.torch.empty((cols, ld_t), dtype=x.dtype, device=x.device) for _ in range(2 if split else 1)]
        self._check(self.lib.c2v_selftest_transpose(self.h, x.data_ptr(), rows, cols, out[0].data_ptr(),
                                                    out[1].data_ptr() if split else None, ld_t, self._stream()))
        return tuple(out) if split else out[0]

    def selftest_gemm_bt(self, A, B, M: int, N: int, K: int, BT, C_out=None):
        """Test hook: C[M,N] = A.B (tf32) with A [M,K] and B [N,K] row-major, and B^T written into BT [K, >= N] by the same
        kernel (c2v_selftest_gemm_bt); returns C."""
        if C_out is None:          # the epilogue stores float4s: 16-byte row pitch
            C_out = self.torch.empty((M, (N + 3) // 4 * 4), dtype=self.torch.float32, device=self.dev)[:, :N]
        out = C_out
        self._check(self.lib.c2v_selftest_gemm_bt(self.h, M, N, K, A.data_ptr(), A.stride(0), B.data_ptr(), B.stride(0),
                                                  out.data_ptr(), out.stride(0), BT.data_ptr(), BT.stride(0), self._stream()))
        return out

    def selftest_target_t(self, lo: bool = False):
        """Test hook: the workspace's K-major copy of the target table that dv reads (c2v_selftest_target_t), as a
        [code_dim, ld] view: the table (tf32) or its transposed high parts (3xTF32); lo: the transposed residuals."""
        off, ld = C.c_size_t(), C.c_size_t()
        self._check(self.lib.c2v_selftest_target_t(self.h, int(lo), C.byref(off), C.byref(ld)))
        n = self.dims.code_dim * ld.value
        return self.workspace[off.value:off.value + 4 * n].view(self.torch.float32).view(self.dims.code_dim, ld.value)

    def selftest_gemm(self, A, B, a_mn: bool, b_mn: bool, M: int, N: int, K: int, bn: int = 192, splits: int = 1,
                      three: bool = False):
        """Test hook: C[M,N] = A.B on the tensor-core (wgmma) path.  A is [M,K] (a_mn False) or [K,M] (True) row-major,
        B is [N,K] (b_mn False) or [K,N] (True); returns C (slices summed on the host side of the test).
        three: as 3xTF32 (operands split on the device first)."""
        torch = self.torch
        out = torch.zeros((max(splits, 1), M, N), dtype=torch.float32, device=self.dev)
        if three:
            (Ah, Al), (Bh, Bl) = self.selftest_split(A), self.selftest_split(B)
            rc = self.lib.c2v_selftest_gemm3(self.h, int(a_mn), int(b_mn), bn, M, N, K, splits, Ah.data_ptr(), Al.data_ptr(),
                                             A.stride(0), Bh.data_ptr(), Bl.data_ptr(), B.stride(0), out.data_ptr(), N,
                                             self._stream())
        else:
            rc = self.lib.c2v_selftest_gemm(self.h, int(a_mn), int(b_mn), bn, M, N, K, splits, A.data_ptr(), A.stride(0),
                                            B.data_ptr(), B.stride(0), out.data_ptr(), N, self._stream())
        if rc < 0:
            self._check(rc)
        return out[:rc].sum(dim=0)

    def selftest_row_sum(self, table_id: int, rows, vals):
        """Test hook for option "deterministic" (c2v_selftest_row_sum): a zeroed copy of table `table_id` (0 = token,
        1 = path) into which row rows[i] receives vals[i] (device int32 [count], float32 [count, embed_dim]), summed by the
        train step's sort + chunked reduce in its documented order.  Returns the table as a device tensor."""
        torch = self.torch
        rows = rows.to(device=self.dev, dtype=torch.int32).contiguous()
        vals = vals.to(device=self.dev, dtype=torch.float32).contiguous()
        n_rows = self.dims.token_vocab if table_id == 0 else self.dims.path_vocab
        out = torch.zeros((n_rows, self.dims.embed_dim), dtype=torch.float32, device=self.dev)
        self._check(self.lib.c2v_selftest_row_sum(self.h, int(table_id), rows.data_ptr(), vals.data_ptr(), int(rows.numel()),
                                                  out.data_ptr(), self._stream()))
        return out

    def selftest_exchange_push(self, tok_rows, tok_vals, path_rows, path_vals):
        """Test hook for option "ordered_exchange" (c2v_selftest_exchange_push): this rank pushes tok_vals[i] for GLOBAL token
        row tok_rows[i] and path_vals[i] for global path row path_rows[i] (int32 [n], float32 [n, embed_dim]) into the
        owners' inboxes, one ordered sum per distinct row.  Barrier, then apply_scatter_inbox() on every rank."""
        torch = self.torch
        i32 = lambda t: torch.as_tensor(t).to(device=self.dev, dtype=torch.int32).contiguous()
        f32 = lambda t: torch.as_tensor(t).to(device=self.dev, dtype=torch.float32).contiguous()
        tr, tv, pr, pv = i32(tok_rows), f32(tok_vals), i32(path_rows), f32(path_vals)
        self._check(self.lib.c2v_selftest_exchange_push(self.h, _ptr(tr), _ptr(tv), int(tr.numel()), _ptr(pr), _ptr(pv),
                                                        int(pr.numel()), self._stream()))
        torch.cuda.current_stream(self.dev).synchronize()       # the lists above may be freed on return

    def phase_stats(self, reset: bool = False) -> Dict[str, Tuple[float, int]]:
        """{phase name: (total device ms, number of timed occurrences)} since the last reset
        (needs set_option("profile", 1)).  Synchronises the device."""
        out = {}
        for i in range(self.lib.c2v_phase_count()):
            ms, n = C.c_double(), C.c_int64()
            self._check(self.lib.c2v_phase_stats(self.h, i, C.byref(ms), C.byref(n), 1 if reset else 0))
            if n.value:
                out[self.lib.c2v_phase_name(i).decode()] = (ms.value, n.value)
        return out

    # ---- parameters -----------------------------------------------------------------------
    def init_params(self, seed: int = 4321, scheme: str = "tensorflow", whole_target_table: bool = False):
        """The reference's initialisers.  scheme "tensorflow" (tensorflow_model.py:205-220,249-250): tables
        U(+-sqrt(3/cols)) (variance_scaling fan_out uniform), TRANSFORM / ATTENTION glorot-uniform.
        scheme "keras" (keras_model.py:46-70, keras_attention_layer.py:29-34): embeddings and the attention
        vector U(+-0.05), both Dense kernels glorot-uniform (the output kernel is [D, |Y|] there).
        Drawn on the device with torch's generator (initialisation is not the hot path).
        whole_target_table: an engine of make_fully_sharded_engine draws the whole target table of global_target_vocab
        rows and keeps its own block, so every rank holds the values a one-GPU engine with the same seed starts from."""
        torch = self.torch
        g = torch.Generator(device=self.dev)
        g.manual_seed(seed)
        d, D, Y = self.dims.embed_dim, self.dims.code_dim, self.dims.target_vocab
        if whole_target_table:
            Y = self.global_target_vocab
        if scheme == "tensorflow":
            lim = {"tok": (3.0 / d) ** 0.5, "path": (3.0 / d) ** 0.5, "tgt": (3.0 / D) ** 0.5,
                   "W": (6.0 / (3 * d + D)) ** 0.5, "a": (6.0 / (D + 1)) ** 0.5}
        elif scheme == "keras":
            lim = {"tok": 0.05, "path": 0.05, "tgt": (6.0 / (D + Y)) ** 0.5, "W": (6.0 / (3 * d + D)) ** 0.5, "a": 0.05}
        else:
            raise ValueError("unknown initialisation scheme: %r" % (scheme,))
        for k in PARAM_NAMES:
            if k == "tgt" and whole_target_table:
                whole = torch.empty((Y, D), dtype=torch.float32, device=self.dev).uniform_(-lim[k], lim[k], generator=g)
                self.params[k].copy_(whole[self.target_row0:self.target_row0 + self.dims.target_vocab])
                continue
            self.params[k].uniform_(-lim[k], lim[k], generator=g)

    def load_params(self, arrays: Dict[str, np.ndarray]):
        torch = self.torch
        for k in PARAM_NAMES:
            src = torch.from_numpy(np.ascontiguousarray(arrays[k], dtype=np.float32))
            if tuple(src.shape) != tuple(self.params[k].shape):
                raise ValueError("parameter %s has shape %s, expected %s" % (k, tuple(src.shape), tuple(self.params[k].shape)))
            self.params[k].copy_(src)

    def sync_tables(self):
        """Lazy Adam: replay deferred updates so the parameter tensors can be read from outside the engine."""
        self._check(self.lib.c2v_sync_tables(self.h, self._stream()))

    def export_params(self) -> Dict[str, np.ndarray]:
        if getattr(self, "table_world", 1) > 1:
            # the token / path tables live in row shards (export_table_shards: this rank's rows); the replicated
            # tensors of the same name are stale and are not handed out
            return {k: self.params[k].detach().cpu().numpy() for k in ("tgt", "W", "a")}
        self.sync_tables()
        return {k: self.params[k].detach().cpu().numpy() for k in PARAM_NAMES}

    def export_grads(self) -> Dict[str, np.ndarray]:
        return {k: self.grads[k].detach().cpu().numpy() for k in PARAM_NAMES}

    def reset_optimizer(self):
        self.sync_tables()
        for d in (self.adam_m, self.adam_v):
            for t in d.values():
                t.zero_()
        self.adam_t = 0
        self.set_option("adam_step_count", 0)

    def to_device(self, arr, dtype):
        torch = self.torch
        if isinstance(arr, torch.Tensor):
            return arr.to(device=self.dev, dtype=dtype).contiguous()
        return torch.from_numpy(np.ascontiguousarray(arr)).to(device=self.dev, dtype=dtype)

    # ---- device-pointer entry points ---------------------------------------------------------
    def forward(self, src, path, tgt, mask, want_attention: bool = True, code_out=None):
        """c2v_forward: (code_vectors [B, D], attention [B, C] or None) as device tensors; code_out: an existing
        [B, D] tensor to write the code vectors into."""
        torch = self.torch
        B, Cn = src.shape
        code = torch.empty((B, self.dims.code_dim), dtype=torch.float32, device=self.dev) if code_out is None else code_out
        attn = torch.empty((B, Cn), dtype=torch.float32, device=self.dev) if want_attention else None
        self._check(self.lib.c2v_forward(self.h, src.data_ptr(), path.data_ptr(), tgt.data_ptr(), mask.data_ptr(),
                                         B, code.data_ptr(), _ptr(attn), self._stream()))
        return code, attn

    def topk(self, code_vec, normalize: bool = False):
        torch = self.torch
        B = code_vec.shape[0]
        k = min(self.dims.top_k, self.dims.target_vocab)
        idx = torch.empty((B, k), dtype=torch.int32, device=self.dev)
        val = torch.empty((B, k), dtype=torch.float32, device=self.dev)
        self._check(self.lib.c2v_topk(self.h, code_vec.data_ptr(), B, idx.data_ptr(), val.data_ptr(),
                                      int(normalize), self._stream()))
        return idx, val

    def loss(self, code_vec, target):
        out = self.torch.empty(1, dtype=self.torch.float32, device=self.dev)
        self._check(self.lib.c2v_loss(self.h, code_vec.data_ptr(), target.data_ptr(), code_vec.shape[0],
                                      out.data_ptr(), self._stream()))
        return out

    def name_scores(self, code_vec, target):
        """c2v_name_scores: (rank [B] int32, logp [B], top1 [B] int32, top1_logp [B]) device tensors -- each example's own
        name (target [B] int32, device) ranked and scored over the whole target vocabulary, in the current math mode."""
        torch = self.torch
        B = code_vec.shape[0]
        if tuple(target.shape) != (B,) or target.dtype != torch.int32 or target.device != self.dev:
            raise ValueError("target must be a [%d] int32 tensor on %s" % (B, self.dev))
        rank = torch.empty(B, dtype=torch.int32, device=self.dev)
        top1 = torch.empty(B, dtype=torch.int32, device=self.dev)
        logp = torch.empty(B, dtype=torch.float32, device=self.dev)
        top1_logp = torch.empty(B, dtype=torch.float32, device=self.dev)
        self._check(self.lib.c2v_name_scores(self.h, code_vec.data_ptr(), target.data_ptr(), B, rank.data_ptr(),
                                             logp.data_ptr(), top1.data_ptr(), top1_logp.data_ptr(), self._stream()))
        return rank, logp, top1, top1_logp

    def train_step(self, src, path, tgt, mask, target, keep: float = 1.0, seed: int = 0, step: int = 0,
                   dropout_mask=None, loss_out=None):
        out = self._loss if loss_out is None else loss_out
        self._check(self.lib.c2v_train_step(self.h, src.data_ptr(), path.data_ptr(), tgt.data_ptr(), mask.data_ptr(),
                                            target.data_ptr(), src.shape[0], float(keep), int(seed), int(step),
                                            _ptr(dropout_mask), out.data_ptr(), self._stream()))
        return out

    def sampled_train_step(self, src, path, tgt, mask, target, sampled, logq_true, logq_sampled, keep: float = 1.0,
                           seed: int = 0, step: int = 0, dropout_mask=None, loss_out=None):
        out = self._loss if loss_out is None else loss_out
        self._check(self.lib.c2v_sampled_train_step(
            self.h, src.data_ptr(), path.data_ptr(), tgt.data_ptr(), mask.data_ptr(), target.data_ptr(),
            src.shape[0], sampled.data_ptr(), sampled.shape[0], logq_true.data_ptr(), logq_sampled.data_ptr(),
            float(keep), int(seed), int(step), _ptr(dropout_mask), out.data_ptr(), self._stream()))
        return out

    def sample_log_uniform(self, target, S: int, seed: int, step: int):
        """c2v_sample_log_uniform: the S unique log-uniform candidates of (seed, step) and the log expected counts of
        them and of target [B] (device int32), as device tensors (sampled int32 [S], logq_true [B], logq_sampled [S],
        num_tries int64 [1]).  The buffers are the engine's own and the next call overwrites them."""
        B, S = int(target.shape[0]), int(S)
        sampled, lq_t, lq_s, tries = self._sampler_buffers(B, S)
        self._check(self.lib.c2v_sample_log_uniform(self.h, S, target.data_ptr(), B, int(seed), int(step), sampled.data_ptr(),
                                                    lq_t.data_ptr(), lq_s.data_ptr(), tries.data_ptr(), self._stream()))
        return sampled, lq_t, lq_s, tries

    def sample_log_uniform_vocab(self, target, S: int, Y: int, seed: int, step: int):
        """c2v_sample_log_uniform_vocab: sample_log_uniform over Y classes (a row-sharded engine passes the global target
        vocabulary, so every rank draws what a one-GPU engine draws for (seed, step)).  Same buffers and results."""
        B, S = int(target.shape[0]), int(S)
        sampled, lq_t, lq_s, tries = self._sampler_buffers(B, S)
        self._check(self.lib.c2v_sample_log_uniform_vocab(self.h, S, int(Y), target.data_ptr(), B, int(seed), int(step),
                                                          sampled.data_ptr(), lq_t.data_ptr(), lq_s.data_ptr(),
                                                          tries.data_ptr(), self._stream()))
        return sampled, lq_t, lq_s, tries

    def _sampler_buffers(self, B: int, S: int):
        torch = self.torch
        buf = getattr(self, "_sampler_out", None)
        if buf is None:          # sized once for the largest call the ABI accepts: S <= 1024, B <= max_batch
            z = lambda n, dt: torch.empty(n, dtype=dt, device=self.dev)
            buf = self._sampler_out = (z(1024, torch.int32), z(self.dims.max_batch, torch.float32), z(1024, torch.float32),
                                       z(1, torch.int64))
        return buf[0][:S], buf[1][:B], buf[2][:S], buf[3]

    def adam_step(self, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, t: Optional[int] = None):
        if t is None:
            self.adam_t += 1
            t = self.adam_t
        else:
            self.adam_t = t
        self._check(self.lib.c2v_adam_step(self.h, lr, beta1, beta2, eps, int(t), self._stream()))

    def arm_target_adam(self, t: int, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8):
        """The next train step's dY epilogue applies Adam step `t` to the target table (c2v_arm_target_adam);
        the following adam_step(t) skips that table.  The target gradient buffer is then not written."""
        self._check(self.lib.c2v_arm_target_adam(self.h, lr, beta1, beta2, eps, int(t)))

    def hint_next_batch(self, src, path, tgt):
        """Device index tensors [B, C] of the batch the next train step will use (c2v_hint_next_batch); the
        caller keeps them alive until that step has been issued."""
        self._check(self.lib.c2v_hint_next_batch(self.h, src.data_ptr(), path.data_ptr(), tgt.data_ptr(), int(src.shape[0])))

    def hint_next_batch_host(self, src, path, tgt):
        """Same from host arrays / pinned tensors (c2v_hint_next_batch_host)."""
        src, path, tgt = (_as_host(x, np.int32) for x in (src, path, tgt))      # pageable sources are staged before the call returns
        self._check(self.lib.c2v_hint_next_batch_host(self.h, _host_ptr(src), _host_ptr(path), _host_ptr(tgt),
                                                      int(src.shape[0]), self._stream()))

    def adam_step_range(self, theta, grad, m, v, t: int, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, zero_grad=False):
        """TF1 Adam on one contiguous slice (the sharded-optimizer path): flat tensors of equal length."""
        n = int(theta.numel())
        assert grad.numel() == n and m.numel() == n and v.numel() == n
        self.adam_t = int(t)
        self._check(self.lib.c2v_adam_step_range(self.h, theta.data_ptr(), grad.data_ptr(), m.data_ptr(), v.data_ptr(),
                                                 n, lr, beta1, beta2, eps, int(t), 1 if zero_grad else 0, self._stream()))

    # ---- phase-split step (fully sharded schedule) ------------------------------------------------
    def context_forward(self, src, path, tgt, mask, code_out, keep=1.0, seed=0, step=0, dropout_mask=None):
        self._check(self.lib.c2v_context_forward(self.h, src.data_ptr(), path.data_ptr(), tgt.data_ptr(), mask.data_ptr(),
                                                 src.shape[0], float(keep), int(seed), int(step), _ptr(dropout_mask),
                                                 code_out.data_ptr(), self._stream()))

    def target_forward(self, code_all, target_all, row_offset, row_max, row_sum, true_logit):
        self._check(self.lib.c2v_target_forward(self.h, code_all.data_ptr(), code_all.shape[0], target_all.data_ptr(),
                                                int(row_offset), row_max.data_ptr(), row_sum.data_ptr(),
                                                true_logit.data_ptr(), self._stream()))

    def lse_combine(self, maxes, sums, true_logit, lse_out, loss_out):
        world, Bt = maxes.shape
        self._check(self.lib.c2v_lse_combine(self.h, maxes.data_ptr(), sums.data_ptr(), world, Bt, true_logit.data_ptr(),
                                             1.0 / Bt, lse_out.data_ptr(), loss_out.data_ptr(), self._stream()))

    def target_backward(self, code_all, lse, target_all, row_offset, dv_partial):
        Bt = code_all.shape[0]
        self._check(self.lib.c2v_target_backward(self.h, code_all.data_ptr(), Bt, lse.data_ptr(), target_all.data_ptr(),
                                                 int(row_offset), 1.0 / Bt, dv_partial.data_ptr(), self._stream()))

    def context_backward(self, src, path, tgt, mask, dv, keep=1.0, seed=0, step=0, dropout_mask=None):
        self._check(self.lib.c2v_context_backward(self.h, src.data_ptr(), path.data_ptr(), tgt.data_ptr(), mask.data_ptr(),
                                                  src.shape[0], float(keep), int(seed), int(step), _ptr(dropout_mask),
                                                  dv.data_ptr(), self._stream()))

    # ---- sampled softmax on a row-sharded target table (fully sharded schedule) -------------------------
    def sampled_pack_rows(self, sampled, target_all, row_offset, neg_rows, true_rows):
        """c2v_sampled_pack_rows: the rows of sampled [S] / target_all [Bt] this engine holds into neg_rows [S, D] /
        true_rows [Bt, D], zeros elsewhere."""
        self._check(self.lib.c2v_sampled_pack_rows(self.h, sampled.data_ptr(), sampled.shape[0], target_all.data_ptr(),
                                                   target_all.shape[0], int(row_offset), neg_rows.data_ptr(),
                                                   true_rows.data_ptr(), self._stream()))

    def sampled_target_step(self, code_vec, target, sampled, logq_true, logq_sampled, neg_rows, true_rows, inv_batch,
                            dv, g_true, g_neg, loss_partial):
        """c2v_sampled_target_step: the sampled head of this rank's examples against the packed rows -> dv [B, D], the
        partial target gradients g_true [B, D] / g_neg [S, D] and loss_partial [1]."""
        self._check(self.lib.c2v_sampled_target_step(
            self.h, code_vec.data_ptr(), code_vec.shape[0], target.data_ptr(), sampled.data_ptr(), sampled.shape[0],
            logq_true.data_ptr(), logq_sampled.data_ptr(), neg_rows.data_ptr(), true_rows.data_ptr(), float(inv_batch),
            dv.data_ptr(), g_true.data_ptr(), g_neg.data_ptr(), loss_partial.data_ptr(), self._stream()))

    def sampled_target_fold(self, g_true_all, g_neg_all, target_all, sampled, row_offset, loss_parts, loss_out):
        """c2v_sampled_target_fold: every rank's partial gradients g_true_all [Bt, D] / g_neg_all [world, S, D] -> this
        engine's target gradient block (cleared first), and loss_out [1] = the sum of loss_parts [world] in rank order."""
        world, S = g_neg_all.shape[0], sampled.shape[0]
        self._check(self.lib.c2v_sampled_target_fold(self.h, g_true_all.data_ptr(), g_neg_all.data_ptr(), world,
                                                     target_all.data_ptr(), target_all.shape[0], sampled.data_ptr(), S,
                                                     int(row_offset), loss_parts.data_ptr(), loss_out.data_ptr(),
                                                     self._stream()))

    # ---- prediction against a row-sharded target table (fully sharded schedule) ------------------------
    def topk_partial(self, code_all, row_offset, k, idx, val, row_max=None, row_sum=None):
        """c2v_topk_partial: this engine's best k target rows for each of the Bt examples of code_all [Bt, D], with global
        ids (local row + row_offset) and raw logits, into idx [Bt, k] (int32) / val [Bt, k]; with row_max / row_sum [Bt],
        the (max, sum exp) of each example's local logits as well (for normalize 2)."""
        self._check(self.lib.c2v_topk_partial(self.h, code_all.data_ptr(), code_all.shape[0], int(row_offset), int(k),
                                              idx.data_ptr(), val.data_ptr(), _ptr(row_max), _ptr(row_sum), self._stream()))

    def topk_merge(self, idx, val, maxes, sums, row0, rows, normalize, idx_out, val_out):
        """c2v_topk_merge: the ranks' candidates idx / val [world, Bt, k] (and maxes / sums [world, Bt], or None unless
        normalize == 2) -> the top k of examples [row0, row0 + rows) into idx_out / val_out [rows, k]."""
        world, Bt, k = idx.shape
        self._check(self.lib.c2v_topk_merge(self.h, idx.data_ptr(), val.data_ptr(), _ptr(maxes), _ptr(sums), world, Bt, k,
                                            int(row0), int(rows), int(normalize), idx_out.data_ptr(), val_out.data_ptr(),
                                            self._stream()))

    # ---- row-sharded embedding tables over peer memory (data-parallel runs) ----------------------
    def apply_scatter_inbox(self):
        """Owner side of the push-based gradient exchange: fold this rank's inbox into its gradient shards (call after
        the cross-rank barrier that follows every rank's backward pass)."""
        self._check(self.lib.c2v_apply_scatter_inbox(self.h, self._stream()))

    def enable_table_sharding(self, group=None, push_grads: bool = False, ordered_exchange: bool = False):
        """Re-homes WORDS_VOCAB / PATHS_VOCAB (+ gradients, Adam slots) as row-interleaved shards: global
        row r -> rank r % world, local row r // world.  Parameter and gradient shards live in
        cudaMalloc'ed memory whose CUDA-IPC handles are exchanged once, so every rank's kernels can
        load rows from, and red.add gradients into, every other rank's shard over NVLink.  The current
        contents of the replicated tables are carried over.  push_grads: gradient rows go through a per-rank inbox instead
        of red.adds; ordered_exchange: through the inbox as sorted per-row sums that the owners fold in rank order (engine
        option "ordered_exchange"), which is what option "deterministic" needs on sharded tables."""
        import torch.distributed as dist
        torch = self.torch
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        if world not in (1, 2, 4, 8):
            raise ValueError("table sharding needs a world size of 1, 2, 4 or 8")
        if self.training and self.get_option("lazy_adam"):
            self.set_option("lazy_adam", 0)          # flushes deferred updates; shards use the dense per-rank Adam
        d = self.dims.embed_dim
        rows = {"tok": (self.dims.token_vocab + world - 1) // world, "path": (self.dims.path_vocab + world - 1) // world}
        own, handles = {}, {}
        self.ordered_exchange = bool(ordered_exchange) and self.training and world > 1
        if self.ordered_exchange:
            self.set_option("ordered_exchange", 1)
        # push_grads also says "an inbox is bound: fold it after the step's barrier", which holds for both routes
        self.push_grads = (bool(push_grads) and self.training and world > 1) or self.ordered_exchange
        if self.push_grads:          # one inbox per rank for the embedding-gradient rows its peers push (c2v_bind_scatter_inbox)
            cd = self.dims.to_c()
            nbytes = self.lib.c2v_scatter_inbox_bytes(C.byref(cd), world)
            ptr, hbuf = _P(), C.create_string_buffer(64)
            rc = self.lib.c2v_ipc_alloc(self.device, nbytes, C.byref(ptr), hbuf)
            if rc != 0:
                raise EngineError(rc, self.lib.c2v_last_error(None).decode())
            own[("inbox", "all")] = ptr.value
            handles[("inbox", "all")] = hbuf.raw
        for role in ("params", "grads"):
            for name in ("tok", "path"):
                ptr, hbuf = _P(), C.create_string_buffer(64)
                rc = self.lib.c2v_ipc_alloc(self.device, rows[name] * d * 4, C.byref(ptr), hbuf)
                if rc != 0:
                    raise EngineError(rc, self.lib.c2v_last_error(None).decode())
                own[(role, name)] = ptr.value
                handles[(role, name)] = hbuf.raw
        gathered = [None] * world
        dist.all_gather_object(gathered, handles, group=group)
        ptrs = {}
        self._ipc_opened = []
        for r in range(world):
            for key in handles:
                if r == rank:
                    ptrs[(r,) + key] = own[key]
                else:
                    p = _P()
                    rc = self.lib.c2v_ipc_open(self.device, gathered[r][key], C.byref(p))
                    if rc != 0:
                        raise EngineError(rc, self.lib.c2v_last_error(None).decode())
                    ptrs[(r,) + key] = p.value
                    self._ipc_opened.append(p.value)
        self._ipc_owned = list(own.values())

        def shards(role):
            st = c2v_table_shards()
            st.world, st.rank = world, rank
            for r in range(world):
                st.tok[r] = ptrs[(r, role, "tok")]
                st.path[r] = ptrs[(r, role, "path")]
            return st

        sp, sg = shards("params"), shards("grads")
        self._check(self.lib.c2v_bind_table_shards(self.h, C.byref(sp), C.byref(sg) if self.training else None, 1.0 / world))
        if self.push_grads:
            arr = (_P * world)(*[ptrs[(r, "inbox", "all")] for r in range(world)])
            self._check(self.lib.c2v_bind_scatter_inbox(self.h, arr, world, rank))
        view = lambda key, name: torch.as_tensor(_DeviceArray(own[key], (rows[name], d)), device=self.dev)
        self.table_world, self.table_rank = world, rank
        self.shard_params = {n: view(("params", n), n) for n in ("tok", "path")}
        self.shard_grads = {n: view(("grads", n), n) for n in ("tok", "path")}
        self.shard_m = {n: torch.zeros((rows[n], d), dtype=torch.float32, device=self.dev) for n in ("tok", "path")}
        self.shard_v = {n: torch.zeros((rows[n], d), dtype=torch.float32, device=self.dev) for n in ("tok", "path")}
        for n in ("tok", "path"):
            mine = self.params[n][rank::world]
            self.shard_params[n][:mine.shape[0]].copy_(mine)
        torch.cuda.synchronize(self.dev)
        dist.barrier(group=group)

    def load_table_shards(self, arrays: Dict[str, np.ndarray]):
        """Fill this rank's shards from full [T, d] / [P, d] host tables."""
        torch = self.torch
        for n in ("tok", "path"):
            mine = np.ascontiguousarray(arrays[n][self.table_rank::self.table_world], dtype=np.float32)
            self.shard_params[n][:mine.shape[0]].copy_(torch.from_numpy(mine))

    def export_table_shards(self) -> Dict[str, np.ndarray]:
        return {n: self.shard_params[n].detach().cpu().numpy() for n in ("tok", "path")}

    # ---- host-buffer entry points ------------------------------------------------------------
    def train_batch_host(self, src, path, tgt, mask, target, keep: float = 1.0, seed: int = 0,
                         lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8) -> float:
        """One reference `sess.run([optimizer, train_loss])` on HOST arrays (numpy or pinned torch
        tensors): H2D copies, train step, Adam, loss read-back -- all inside the C-ABI call."""
        loss = np.zeros(1, dtype=np.float32)
        B = int(src.shape[0])
        src, path, tgt, target = (_as_host(x, np.int32) for x in (src, path, tgt, target))
        mask = _as_host(mask, np.float32)
        self._check(self.lib.c2v_train_batch_host(
            self.h, _host_ptr(src), _host_ptr(path), _host_ptr(tgt), _host_ptr(mask), _host_ptr(target), B,
            float(keep), int(seed), int(self.adam_t + 1), lr, beta1, beta2, eps, loss.ctypes.data, self._stream()))
        self.adam_t += 1          # only once the step went through: a failed call leaves host and engine counters in step
        return float(loss[0])

    def train_batch_async(self, src, path, tgt, mask, target, rows: int, loss_out, upload_done=None, keep: float = 1.0,
                          seed: int = 0, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8):
        """c2v_train_batch_async on PINNED torch tensors (first `rows` rows): the upload runs on the engine's copy stream,
        the step is queued behind it, nothing is waited for.  loss_out: pinned float32 tensor of one element; upload_done:
        torch.cuda.Event recorded when the inputs have left the host buffers."""
        for x in (src, path, tgt, mask, target, loss_out):
            if not x.is_pinned():
                raise ValueError("c2v_train_batch_async needs page-locked host tensors")
        ev = None
        if upload_done is not None:
            upload_done.record(self.torch.cuda.current_stream(self.dev))      # forces creation of the cudaEvent_t; re-recorded by the engine
            ev = upload_done.cuda_event
        self._check(self.lib.c2v_train_batch_async(
            self.h, src.data_ptr(), path.data_ptr(), tgt.data_ptr(), mask.data_ptr(), target.data_ptr(), int(rows),
            float(keep), int(seed), int(self.adam_t + 1), lr, beta1, beta2, eps, loss_out.data_ptr(), ev, self._stream()))
        self.adam_t += 1

    def predict_batch_host(self, src, path, tgt, mask, normalize: bool = False, want_code: bool = True,
                           want_attention: bool = True):
        B, Cn = int(src.shape[0]), int(src.shape[1])
        src, path, tgt = (_as_host(x, np.int32) for x in (src, path, tgt))
        mask = _as_host(mask, np.float32)
        k = min(self.dims.top_k, self.dims.target_vocab)
        idx = np.empty((B, k), dtype=np.int32)
        val = np.empty((B, k), dtype=np.float32)
        code = np.empty((B, self.dims.code_dim), dtype=np.float32) if want_code else None
        attn = np.empty((B, Cn), dtype=np.float32) if want_attention else None
        self._check(self.lib.c2v_predict_batch_host(
            self.h, _host_ptr(src), _host_ptr(path), _host_ptr(tgt), _host_ptr(mask), B, int(normalize),
            idx.ctypes.data, val.ctypes.data, None if code is None else code.ctypes.data,
            None if attn is None else attn.ctypes.data, self._stream()))
        return idx, val, code, attn


_TORCH_DTYPE_NAMES = {np.dtype(np.int32): "torch.int32", np.dtype(np.float32): "torch.float32"}


def _as_host(a, dtype):
    """numpy arrays are made contiguous/typed (no copy when already so); torch CPU tensors pass through, but only
    with the element type the C entry point reads -- an int64 index tensor read as int32 would index the tables
    out of range without any error."""
    if isinstance(a, np.ndarray):
        return np.ascontiguousarray(a, dtype=dtype)
    if hasattr(a, "dtype") and hasattr(a, "data_ptr"):
        want = _TORCH_DTYPE_NAMES[np.dtype(dtype)]
        if str(a.dtype) != want:
            raise TypeError("host tensor has dtype %s, the engine reads %s" % (a.dtype, want))
    return a


def _host_ptr(a) -> int:
    """Address of a contiguous host buffer: numpy array or (pinned) CPU torch tensor."""
    if isinstance(a, np.ndarray):
        if not a.flags["C_CONTIGUOUS"]:
            raise ValueError("host buffer must be C-contiguous")
        return a.ctypes.data
    if hasattr(a, "data_ptr"):
        if a.device.type != "cpu" or not a.is_contiguous():
            raise ValueError("host buffer must be a contiguous CPU tensor")
        return a.data_ptr()
    raise TypeError("unsupported host buffer type %r" % type(a))


# ---- CRC-32C of device tensors (tf_bundle.py, DESIGN.md §6k) ----------------------------------------------------------
def crc32c_rows(x, rows: int, row_bytes: int, row_stride: int, out) -> None:
    """out (device int32 [>= rows], read as uint32) = the CRC-32C of each of the `rows` rows of row_bytes bytes of the
    device tensor x, row r at byte r * row_stride of it; queued on the current stream."""
    import torch
    lib = load_library()
    rc = lib.c2v_crc32c_rows(x.data_ptr() if rows else None, int(rows), int(row_bytes), int(row_stride), out.data_ptr(),
                             torch.cuda.current_stream(out.device).cuda_stream)
    if rc != 0:
        raise EngineError(rc, lib.c2v_last_error(None).decode())


def crc32c_combine(crcs, n: int, seg_bytes: int, out) -> None:
    """out[0] (device int32, read as uint32) = the CRC-32C of n segments of seg_bytes bytes whose CRCs are crcs[0, n)
    (device int32); queued on the current stream."""
    import torch
    lib = load_library()
    rc = lib.c2v_crc32c_combine(crcs.data_ptr() if n else None, int(n), int(seg_bytes), out.data_ptr(),
                                torch.cuda.current_stream(out.device).cuda_stream)
    if rc != 0:
        raise EngineError(rc, lib.c2v_last_error(None).decode())


def tensor_crc32c(x, rows: int, row_bytes: int, out) -> None:
    """out[0] = the CRC-32C of the first rows * row_bytes bytes of the contiguous device tensor x, as `rows` rows
    checked in parallel and combined; queued on the current stream."""
    import torch
    row_crc = torch.empty(max(int(rows), 1), dtype=torch.int32, device=x.device)
    crc32c_rows(x, rows, row_bytes, row_bytes, row_crc)
    crc32c_combine(row_crc, rows, row_bytes, out)


# ---- the Keras output kernel's transpose (keras_ckpt.py, DESIGN.md §6l) -----------------------------------------------
def rows_to_cols(src, k: int, Y: int, dst, col0: int) -> None:
    """dst[y, col0 + i] = src[i * Y + y] for i < k, y < Y, bit for bit: k file rows of a [D, Y] kernel (the contiguous
    device tensor src) into columns of the contiguous device table dst [Y, ld]; queued on the current stream."""
    import torch
    lib = load_library()
    rc = lib.c2v_rows_to_cols(src.data_ptr(), int(k), int(Y), dst.data_ptr(), int(dst.shape[-1]), int(col0),
                              torch.cuda.current_stream(dst.device).cuda_stream)
    if rc != 0:
        raise EngineError(rc, lib.c2v_last_error(None).decode())


def cols_to_rows(src, col0: int, k: int, Y: int, dst) -> None:
    """dst[i * Y + y] = src[y, col0 + i] for i < k, y < Y, bit for bit: the reverse of rows_to_cols; queued on the current
    stream."""
    import torch
    lib = load_library()
    rc = lib.c2v_cols_to_rows(src.data_ptr(), int(src.shape[-1]), int(col0), int(k), int(Y), dst.data_ptr(),
                              torch.cuda.current_stream(dst.device).cuda_stream)
    if rc != 0:
        raise EngineError(rc, lib.c2v_last_error(None).decode())
