#!/usr/bin/env python
"""Keras checkpoint rates on one H100 (DESIGN.md §6l): prints one JSON line per measurement.

  * A java14m-shaped model (T = 1,301,137, P = 911,418, Y = 261,246, d = 128, D = 384) with its Adam slots is saved in
    the reference Keras backend's format (C2V_SAVE_FORMAT=keras: `__entire-model/ckpt-N` with the optimizer, and
    `__only-weights`) and as a TensorFlow bundle (C2V_SAVE_FORMAT=tf) in a temporary directory, each save timed; then each
    is loaded best of three from the page cache, alternating the formats: into an inference engine (the weights, 1.53 GB)
    and into a training engine (weights and Adam slots, 4.6 GB).  Both loads include their CRC-32C checks; the Keras
    load also transposes the [D, Y] output kernel (and its slots) on the GPU.
  * c2v_rows_to_cols and c2v_cols_to_rows alone over the whole [384, 261,246] kernel: CUDA events around 20 calls, in
    GB/s (bytes read + written) against the 3.35 TB/s HBM3 bound of the H100 SXM data sheet.
The card's name and power limit are read in the same run and printed with the numbers."""
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

JAVA14M = dict(token_vocab=1301137, path_vocab=911418, target_vocab=261246, embed_dim=128, code_dim=384, max_contexts=200,
               max_batch=64, top_k=10)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def _model(engine, save_format, release=False):
    """A Code2VecModel around `engine` with only what its checkpoint methods use."""
    from code2vec_b200.b200_model import Code2VecModel

    class Cfg:
        RELEASE, MAX_TO_KEEP = release, 10
    m = Code2VecModel.__new__(Code2VecModel)
    m.engine, m.world, m.rank, m._save_format, m.config = engine, 1, 0, save_format, Cfg()
    return m


def _timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    import torch
    from code2vec_b200.engine import EngineDims, PathAttentionEngine, cols_to_rows, rows_to_cols
    print(json.dumps(dict(what="card", card=card())), flush=True)
    tmp = tempfile.mkdtemp(prefix="c2v_keras_rate_")
    try:
        e = PathAttentionEngine(EngineDims(**JAVA14M), device=0, training=True)
        e.init_params()
        e.adam_t = 1234
        x = os.path.join(tmp, "k")
        bundle = os.path.join(tmp, "b")
        saves = [("keras entire model (weights + Adam)", lambda: _model(e, "keras")._save_inner_model(x)),
                 ("keras weights", lambda: _model(e, "keras", release=True)._save_inner_model(x)),
                 ("tf bundle (weights + Adam)", lambda: _model(e, "tf")._save_inner_model(bundle)),
                 ("tf bundle weights", lambda: _model(e, "tf")._save_inner_model(bundle + ".release", release=True))]
        for what, fn in saves:
            print(json.dumps(dict(what="save", format=what, s=round(_timed(fn), 3))), flush=True)
        e.close()
        ckpt = os.path.join(x + "__entire-model", "ckpt-0")
        for training in (False, True):
            eng = PathAttentionEngine(EngineDims(**JAVA14M), device=0, training=training)
            m = _model(eng, "c2v_b200")
            loads = {"keras": (lambda: m._read_keras(ckpt)) if training else (lambda: m._read_keras(x + "__only-weights")),
                     "tf": (lambda: m._read_bundle(bundle)) if training else (lambda: m._read_bundle(bundle + ".release"))}
            best = {k: float("inf") for k in loads}
            for _ in range(3):
                for fmt, fn in loads.items():             # alternated, so both see the same page cache and clocks
                    best[fmt] = min(best[fmt], _timed(fn))
            nbytes = sum(t.numel() * 4 for g in ((eng.params, eng.adam_m, eng.adam_v) if training else (eng.params,))
                         for t in g.values())
            for fmt, s in best.items():
                print(json.dumps(dict(what="load", format=fmt, tensors="weights + Adam" if training else "weights",
                                      GB=round(nbytes / 1e9, 3), best_of_3_s=round(s, 3),
                                      GB_per_s=round(nbytes / 1e9 / s, 2))), flush=True)
            if training:
                tgt = eng.params["tgt"]
                Y, D = tgt.shape
                chunk = torch.empty(D * Y, dtype=torch.float32, device=eng.dev)
                for name, fn in (("c2v_rows_to_cols", lambda: rows_to_cols(chunk, D, Y, tgt, 0)),
                                 ("c2v_cols_to_rows", lambda: cols_to_rows(tgt, 0, D, Y, chunk))):
                    for _ in range(3):
                        fn()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    for _ in range(20):
                        fn()
                    b.record()
                    torch.cuda.synchronize()
                    ms = a.elapsed_time(b) / 20
                    gbs = 2 * D * Y * 4 / 1e9 / (ms / 1e3)
                    print(json.dumps(dict(what=name, k=D, Y=Y, ms=round(ms, 3), GB_per_s=round(gbs, 1),
                                          share_of_hbm_bound=round(gbs / 3350, 3))), flush=True)
            eng.close()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
