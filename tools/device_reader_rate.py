#!/usr/bin/env python
"""The training reader alone, on the GPU and on the host: lines/s of DeviceBatchReader (file -> device batches, the
device synchronised at the end) and of PathContextReader's native path (file -> host batches), over the synthetic
java14m-shaped `.c2v` file of tools/reader_rate.py, with that tool's vocabulary sizes and with java14m's (1.3 M tokens,
911 K paths, 261 K targets).  Also reports the device memory the reader holds, the card's name and power limit and the
host's core count.  `--profile` runs one more device pass under torch.profiler and reports the reader's kernel time per
batch.  Prints one JSON line per vocabulary size.  Writes only to a temporary directory."""
import json
import os
import pickle
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def _dataset(tmp, n_lines, C, n_tok, n_path, n_tgt):
    prefix = os.path.join(tmp, "syn%d" % n_tok)
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
    return prefix


def run(tmp, n_tok, n_path, n_tgt, n_lines=65536, C=200, threads=16, batch=1024, profile=False):
    import torch
    from code2vec_b200.b200_model import _TrainInputFormer
    from code2vec_b200.config import Config
    from code2vec_b200.device_reader import DeviceBatchReader
    from code2vec_b200.path_context_reader import EstimatorAction, PathContextReader
    from code2vec_b200.vocabularies import Code2VecVocabs
    prefix = _dataset(tmp, n_lines, C, n_tok, n_path, n_tgt)
    cfg = Config(set_defaults=True)
    cfg.VERBOSE_MODE = 0
    cfg.DL_FRAMEWORK = "b200"
    cfg.TRAIN_DATA_PATH_PREFIX = prefix
    cfg.NUM_TRAIN_EPOCHS = 1
    cfg.TRAIN_BATCH_SIZE = batch
    cfg.READER_NUM_PARALLEL_BATCHES = threads
    cfg.MAX_TOKEN_VOCAB_SIZE, cfg.MAX_PATH_VOCAB_SIZE, cfg.MAX_TARGET_VOCAB_SIZE = n_tok, n_path, n_tgt
    vocabs = Code2VecVocabs(cfg)
    dev = torch.device("cuda", 0)
    reader = lambda: PathContextReader(vocabs=vocabs, model_input_tensors_former=_TrainInputFormer(), config=cfg,
                                       estimator_action=EstimatorAction.Train, shuffle_seed=1)
    device_rates, host_rates, held, setup_s, batches = [], [], 0, [], 0
    for _ in range(3):                                   # alternating; the first pass also warms the page cache
        t0 = time.time()
        rows = sum(int(b[0].shape[0]) for b in reader().get_dataset())
        host_rates.append(rows / (time.time() - t0))
        t0 = time.time()
        dr = DeviceBatchReader(reader(), dev)
        torch.cuda.synchronize()
        setup_s.append(time.time() - t0)                 # vocabulary upload and handle creation
        t0 = time.time()
        rows = batches = 0
        for b in dr:
            b.wait()
            rows += b.rows
            batches += 1
            b.release()
        torch.cuda.synchronize()
        device_rates.append(rows / (time.time() - t0))
        held = dr.device_bytes()
        dr.close()
    out = {"what": "training reader alone: DeviceBatchReader (file -> device batches) vs PathContextReader (file -> host "
                   "batches)", "card_and_power_limit": _card(), "host_cores": os.cpu_count(), "lines": n_lines,
           "contexts_per_line": C, "batch": batch, "host_reader_threads": threads,
           "vocab_words": [n_tok, n_path, n_tgt], "device_lines_per_s": [round(r) for r in device_rates],
           "host_lines_per_s": [round(r) for r in host_rates], "best_device_lines_per_s": round(max(device_rates)),
           "best_host_lines_per_s": round(max(host_rates)), "device_reader_setup_s": [round(s, 2) for s in setup_s],
           "device_bytes_held": held, "batches": batches}
    if profile:
        from torch.profiler import ProfilerActivity, profile as prof
        dr = DeviceBatchReader(reader(), dev)
        with prof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
            for b in dr:
                b.wait()
                b.release()
            torch.cuda.synchronize()
        dr.close()
        kernels = {}
        for e in p.key_averages():
            if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0) > 0:
                us = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
                if us > 0:
                    kernels[e.key[:60]] = round(us / max(batches, 1), 1)
        out["profile_us_per_batch"] = dict(sorted(kernels.items(), key=lambda kv: -kv[1])[:14])
    return out


def main():
    tmp = tempfile.mkdtemp()
    try:
        prof = "--profile" in sys.argv
        print(json.dumps(run(tmp, 200000, 150000, 30000, profile=prof)), flush=True)         # tools/reader_rate.py's sizes
        print(json.dumps(run(tmp, 1300000, 911000, 261000, profile=prof)), flush=True)       # java14m's
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
