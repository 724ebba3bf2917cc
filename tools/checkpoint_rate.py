#!/usr/bin/env python
"""Checkpoint load rates on one H100 (DESIGN.md §6k): prints one JSON line per measurement.

  * A java14m-shaped model (T = 1,301,137, P = 911,418, Y = 261,246, d = 128, D = 384) with its Adam slots is saved once
    as a TensorFlow bundle (C2V_SAVE_FORMAT=tf) and once as a .c2v_b200 checkpoint in a temporary directory, then each
    is loaded best of three from the page cache: into an inference engine (the weights, 1.53 GB: what a release
    holds) and into a training engine (weights and Adam slots, 4.6 GB).  The bundle load includes its CRC-32C checks.
  * c2v_crc32c_rows alone over the token table (512-byte rows): CUDA events around 20 calls, in GB/s against the
    3.35 TB/s HBM3 bound of the H100 SXM data sheet.
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


def _model(engine, save_format):
    """A Code2VecModel around `engine` with only what its checkpoint methods use."""
    from code2vec_b200.b200_model import Code2VecModel
    m = Code2VecModel.__new__(Code2VecModel)
    m.engine, m.world, m.rank, m._save_format = engine, 1, 0, save_format
    return m


def main():
    import torch
    from code2vec_b200.engine import EngineDims, PathAttentionEngine, crc32c_rows
    print(json.dumps(dict(what="card", card=card())), flush=True)
    tmp = tempfile.mkdtemp(prefix="c2v_ckpt_rate_")
    try:
        e = PathAttentionEngine(EngineDims(**JAVA14M), device=0, training=True)
        e.init_params()
        e.adam_t = 1234
        bundle, c2v = os.path.join(tmp, "b"), os.path.join(tmp, "c")
        for path, fmt in ((bundle, "tf"), (c2v, "c2v_b200")):
            t0 = time.perf_counter()
            _model(e, fmt)._save_inner_model(path)
            torch.cuda.synchronize()
            print(json.dumps(dict(what="save", format=fmt, s=round(time.perf_counter() - t0, 3))), flush=True)
        e.close()
        for training in (False, True):
            eng = PathAttentionEngine(EngineDims(**JAVA14M), device=0, training=training)
            m_tf, m_c2v = _model(eng, "tf"), _model(eng, "c2v_b200")
            loads = {"tf": lambda: m_tf._read_bundle(bundle), "c2v_b200": lambda: m_c2v._read_checkpoint(c2v + ".c2v_b200")}
            best = {k: float("inf") for k in loads}
            for _ in range(3):
                for fmt, fn in loads.items():             # alternated, so both see the same page cache and clocks
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    best[fmt] = min(best[fmt], time.perf_counter() - t0)
            nbytes = sum(t.numel() * 4 for g in ((eng.params, eng.adam_m, eng.adam_v) if training else (eng.params,))
                         for t in g.values())
            for fmt, s in best.items():
                print(json.dumps(dict(what="load", format=fmt, tensors="weights + Adam" if training else "weights",
                                      GB=round(nbytes / 1e9, 3), best_of_3_s=round(s, 3),
                                      GB_per_s=round(nbytes / 1e9 / s, 2))), flush=True)
            if training:
                tok = eng.params["tok"]
                rows, row_bytes = tok.shape[0], tok.shape[1] * 4
                out = torch.empty(rows, dtype=torch.int32, device=eng.dev)
                for _ in range(3):
                    crc32c_rows(tok, rows, row_bytes, row_bytes, out)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(20):
                    crc32c_rows(tok, rows, row_bytes, row_bytes, out)
                b.record()
                torch.cuda.synchronize()
                ms = a.elapsed_time(b) / 20
                gbs = rows * row_bytes / 1e9 / (ms / 1e3)
                print(json.dumps(dict(what="c2v_crc32c_rows", rows=rows, row_bytes=row_bytes, ms=round(ms, 3),
                                      GB_per_s=round(gbs, 1), share_of_hbm_bound=round(gbs / 3350, 3))), flush=True)
            eng.close()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
