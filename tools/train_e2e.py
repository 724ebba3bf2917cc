#!/usr/bin/env python
"""End-to-end check of the whole user path on one GPU: a synthetic java14m-shaped `.c2v` file ->
PathContextReader (native tensoriser, prefetch thread) -> Code2VecModel.train() -> C-ABI engine.
Prints one JSON line with examples/s and path-contexts/s as the reference's own progress line would
report them (tensorflow_model.py:424-430).  Not part of bench.py: text parsing is host work outside
the hot path; this measures that the batcher keeps the GPU fed."""
import json
import os
import pickle
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main(n_lines=131072, C=200, n_tok=200000, n_path=150000, n_tgt=30000, threads=16, epochs=4):
    from code2vec_b200.b200_model import Code2VecModel
    from code2vec_b200.config import Config
    tmp = tempfile.mkdtemp()
    prefix = os.path.join(tmp, "syn")
    rng = np.random.default_rng(0)
    toks = ["tok%d" % i for i in range(n_tok)]
    paths = [str(1000003 * i % 2147483647 - 1073741823) for i in range(n_path)]
    tgts = ["do|thing%d" % i for i in range(n_tgt)]
    t0 = time.time()
    with open(prefix + ".train.c2v", "w") as f:
        for _ in range(n_lines):
            k = int(rng.integers(60, C + 1))
            s = rng.integers(0, n_tok, size=(k, 2))
            p = rng.integers(0, n_path, size=k)
            f.write(" ".join([tgts[int(rng.integers(0, n_tgt))]] +
                             ["%s,%s,%s" % (toks[a], paths[b], toks[c]) for (a, c), b in zip(s, p)] + [""] * (C - k)) + "\n")
    with open(prefix + ".dict.c2v", "wb") as f:
        for words in (toks, paths, tgts):
            pickle.dump({w: 2 for w in words}, f)
        pickle.dump(n_lines, f)
    gen_s = time.time() - t0
    cfg = Config(set_defaults=True)
    cfg.VERBOSE_MODE = 0
    cfg.DL_FRAMEWORK = "b200"
    cfg.TRAIN_DATA_PATH_PREFIX = prefix
    cfg.NUM_TRAIN_EPOCHS = epochs
    cfg.SAVE_EVERY_EPOCHS = 1000
    cfg.READER_NUM_PARALLEL_BATCHES = threads
    cfg.SHUFFLE_BUFFER_SIZE = 4096
    cfg.MAX_TOKEN_VOCAB_SIZE, cfg.MAX_PATH_VOCAB_SIZE, cfg.MAX_TARGET_VOCAB_SIZE = n_tok, n_path, n_tgt
    model = Code2VecModel(cfg)
    import torch
    stamps = []
    # the training loop uploads batches through the pinned ring and launches steps asynchronously (step_ring); with
    # C2V_BATCH_RING=0 it calls the synchronous step_host instead.  Either way the host time at which step k was issued is
    # recorded: the ring bounds how far the host can run ahead of the GPU (10 slots), so over hundreds of steps the issue
    # rate is the execution rate.
    # with C2V_DEVICE_READER=1 the loop feeds device slots to step_device instead; with C2V_NUM_SAMPLED=<S> every route
    # steps through step_sampled
    for name in ("step_host", "step_ring", "step_device", "step_sampled"):
        inner = getattr(model.trainer, name)

        def stamped(*a, _inner=inner, **k):
            out = _inner(*a, **k)
            stamps.append(time.time())
            return out
        setattr(model.trainer, name, stamped)
    torch.cuda.synchronize()
    t0 = time.time()
    model.train()
    torch.cuda.synchronize()
    dt = time.time() - t0
    skip = max(len(stamps) // 4, 1)    # steady state: after the reader threads and the prefetch queue have filled
    steady = (len(stamps) - 1 - skip) * cfg.TRAIN_BATCH_SIZE * C / max(stamps[-1] - stamps[skip], 1e-9)
    size_mb = os.path.getsize(prefix + ".train.c2v") / 1e6
    print(json.dumps({"what": "Code2VecModel.train() end to end (file -> native reader -> engine)", "examples": n_lines * epochs, "epochs": epochs,
                      "contexts_per_example": C, "seconds": round(dt, 3), "examples_per_s": round(n_lines * epochs / dt, 1),
                      "path_contexts_per_s": round(n_lines * epochs * C / dt, 1),
                      "steady_state_path_contexts_per_s": round(steady, 1), "batches": len(stamps), "file_MB": round(size_mb, 1),
                      "text_MB_per_s": round(size_mb * epochs / dt, 1), "reader_threads": threads, "host_cores": os.cpu_count(),
                      "reader": "device" if model._device_reader else "host", "num_sampled": model._num_sampled,
                      "target_vocab": model.vocabs.target_vocab.size,
                      "batch_ring": os.environ.get("C2V_BATCH_RING", "1") != "0" and not model._device_reader,
                      "h2d_bytes_total": int(getattr(model, "h2d_bytes", 0)),
                      "dataset_generation_s": round(gen_s, 1)}))
    model.close_session()


if __name__ == "__main__":
    main(threads=int(sys.argv[1]) if len(sys.argv) > 1 else 16)
