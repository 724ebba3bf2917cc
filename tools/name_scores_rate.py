#!/usr/bin/env python
"""Code2VecModel.score_names (`--score_names`, DESIGN.md §6n) at java14m's model dims (1,301,137 tokens, 911,418 paths,
261,246 targets, d = 128, D = 384, C = 200) with seeded parameters, over the synthetic java14m-shaped test file that
tools/eval_rate.py builds (65,536 lines by default).

  1. c2v_name_scores on one 1,024-row batch of code vectors, in tf32 and 3xTF32: GPU ms per call from CUDA events over
     --steps calls in each of --windows windows (median, min, max), then one profiled window split by engine phase
     (split = the 3xTF32 operand split, logits = the logits GEMM writing the slab, name_rank = the one pass over it).  The
     name_rank phase's slab read (B x Y x 4 bytes) over its time gives its achieved bandwidth.
  2. score_names end to end (host reader, forward, logits + rank, copy-back), rows/s, best of --passes after a warm-up.
Prints one JSON line with the card's name and power limit.  Writes only to a temporary directory."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from eval_rate import JAVA14M, _card, _dataset  # noqa: E402


def kernel_times(e, B, steps, windows):
    import torch
    g = torch.Generator(device=e.dev).manual_seed(3)
    v = 3.0 * torch.randn((B, e.dims.code_dim), generator=g, device=e.dev)
    y = torch.randint(0, e.dims.target_vocab, (B,), generator=g, device=e.dev, dtype=torch.int32)
    out = {}
    for math_mode, name in ((1, "tf32"), (2, "3xtf32")):
        e.set_option("math_mode", math_mode)
        for _ in range(3):
            e.name_scores(v, y)
        ms = []
        for _ in range(windows):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                e.name_scores(v, y)
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b) / steps)
        e.set_option("profile", 1)
        e.phase_stats(reset=True)
        for _ in range(steps):
            e.name_scores(v, y)
        ph = e.phase_stats(reset=True)
        e.set_option("profile", 0)
        per = {k: round(t / steps, 4) for k, (t, _) in sorted(ph.items())}
        slab = B * e.dims.target_vocab * 4
        t = np.array(ms)
        out[name] = dict(ms_per_batch_median=round(float(np.median(t)), 4), ms_per_batch_min=round(float(t.min()), 4),
                         ms_per_batch_max=round(float(t.max()), 4), phase_ms_per_batch=per,
                         name_rank_slab_read_TBps=round(slab / (per["name_rank"] * 1e-3) / 1e12, 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=65536)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    args = ap.parse_args()
    import torch
    from code2vec_b200.b200_model import Code2VecModel
    from code2vec_b200.config import Config
    tmp = tempfile.mkdtemp(prefix="c2v_name_scores_rate_")
    try:
        T, P, Y = JAVA14M
        prefix = _dataset(tmp, args.lines, 200, T - 2, P - 2, Y - 1)
        cfg = Config(set_defaults=True)
        cfg.VERBOSE_MODE = 0
        cfg.DL_FRAMEWORK = "b200"
        cfg.TRAIN_DATA_PATH_PREFIX = prefix                  # the vocabularies come from its dictionary; nothing trains
        cfg.MAX_TOKEN_VOCAB_SIZE, cfg.MAX_PATH_VOCAB_SIZE, cfg.MAX_TARGET_VOCAB_SIZE = T, P, Y
        os.environ.setdefault("C2V_SEED", "7")
        model = Code2VecModel(cfg)
        dims = model.engine.dims
        try:
            kernels = kernel_times(model.engine, cfg.TEST_BATCH_SIZE, args.steps, args.windows)
            data = prefix + ".test.c2v"
            model.score_names(data)                          # warm-up: page cache, reader
            secs, ref = [], None
            for _ in range(args.passes):
                torch.cuda.synchronize()
                t0 = time.time()
                res = model.score_names(data)
                torch.cuda.synchronize()
                secs.append(time.time() - t0)
                if ref is None:
                    ref = res
                assert all(np.array_equal(a, b) for a, b in zip(res[1:], ref[1:])), "passes differ"
            rows = len(ref[0])
            out = {"what": "c2v_name_scores per 1,024-row batch (logits + rank) and score_names end to end",
                   "card_and_power_limit": _card(), "host_cores": os.cpu_count(), "lines": args.lines, "rows": rows,
                   "dims": {"tokens": dims.token_vocab, "paths": dims.path_vocab, "targets": dims.target_vocab,
                            "d": dims.embed_dim, "D": dims.code_dim, "C": dims.max_contexts, "batch": cfg.TEST_BATCH_SIZE},
                   "kernel": kernels, "score_names_s": [round(s, 3) for s in secs],
                   "score_names_rows_per_s": round(rows / min(secs)),
                   "score_names_math": {1: "tf32", 2: "3xtf32", 0: "fp32"}[model._math_eval]}
            print(json.dumps(out))
        finally:
            model.close_session()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
