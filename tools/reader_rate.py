#!/usr/bin/env python
"""The training reader alone (no GPU): lines/s of PathContextReader over a synthetic java14m-shaped `.c2v` file, with the
native tensoriser, the shuffle pool and batches of TRAIN_BATCH_SIZE rows, as Code2VecModel.train() drives it.

On several GPUs every rank runs this same reader over the whole training file and keeps its slice of each global batch
(DESIGN.md §6c), so this rate bounds the multi-GPU step rate: steps/s <= lines/s / TRAIN_BATCH_SIZE.  Prints one JSON
line.  Writes only to a temporary directory."""
import json
import os
import pickle
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main(n_lines=65536, C=200, n_tok=200000, n_path=150000, n_tgt=30000, threads=16, batch=1024):
    from code2vec_b200.b200_model import _TrainInputFormer
    from code2vec_b200.config import Config
    from code2vec_b200.path_context_reader import EstimatorAction, PathContextReader
    from code2vec_b200.vocabularies import Code2VecVocabs
    tmp = tempfile.mkdtemp()
    try:
        prefix = os.path.join(tmp, "syn")
        rng = np.random.default_rng(0)
        toks = ["tok%d" % i for i in range(n_tok)]
        paths = [str(1000003 * i % 2147483647 - 1073741823) for i in range(n_path)]
        tgts = ["do|thing%d" % i for i in range(n_tgt)]
        with open(prefix + ".train.c2v", "w") as f:
            for _ in range(n_lines):
                k = int(rng.integers(60, C + 1))
                s = rng.integers(0, n_tok, size=(k, 2))
                p = rng.integers(0, n_path, size=k)
                f.write(" ".join([tgts[int(rng.integers(0, n_tgt))]] + ["%s,%s,%s" % (toks[a], paths[b], toks[c])
                                                                         for (a, c), b in zip(s, p)] + [""] * (C - k)) + "\n")
        with open(prefix + ".dict.c2v", "wb") as f:
            for words in (toks, paths, tgts):
                pickle.dump({w: 2 for w in words}, f)
            pickle.dump(n_lines, f)
        cfg = Config(set_defaults=True)
        cfg.VERBOSE_MODE = 0
        cfg.DL_FRAMEWORK = "b200"
        cfg.TRAIN_DATA_PATH_PREFIX = prefix
        cfg.NUM_TRAIN_EPOCHS = 1
        cfg.TRAIN_BATCH_SIZE = batch
        cfg.READER_NUM_PARALLEL_BATCHES = threads
        cfg.MAX_TOKEN_VOCAB_SIZE, cfg.MAX_PATH_VOCAB_SIZE, cfg.MAX_TARGET_VOCAB_SIZE = n_tok, n_path, n_tgt
        vocabs = Code2VecVocabs(cfg)
        rates = []
        for _ in range(3):                   # the first pass also warms the page cache
            reader = PathContextReader(vocabs=vocabs, model_input_tensors_former=_TrainInputFormer(), config=cfg,
                                       estimator_action=EstimatorAction.Train, shuffle_seed=1)
            t0 = time.time()
            rows = sum(int(b[0].shape[0]) for b in reader.get_dataset())
            rates.append(rows / (time.time() - t0))
        print(json.dumps({"what": "PathContextReader train pass alone (native tensoriser, shuffle pool)", "lines": n_lines,
                          "contexts_per_line": C, "batch": batch, "reader_threads": threads, "host_cores": os.cpu_count(),
                          "native": bool(reader._native_ready()), "lines_per_s": [round(r) for r in rates],
                          "best_lines_per_s": round(max(rates)), "steps_per_s_bound": round(max(rates) / batch, 1)}))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
