#!/usr/bin/env python
"""Seconds from `Code2VecModel(config)` to the end of the first training step when fine-tuning a java14m-sized model,
with and without C2V_EXTEND_VOCAB=1 (DESIGN.md §6m); prints one JSON line per measurement.

A temporary directory gets a java14m-shaped model (T = 1,301,137, P = 911,418, Y = 261,246, d = 128, D = 384) with
its Adam slots, saved as a TensorFlow bundle as the published model is, beside a dictionaries.bin of synthetic words,
and a dataset whose `.dict.c2v` holds 200,000 tokens, 100,000 paths and 50,000 method names the model lacks (plus a few
it has) and whose training file is one batch of 64 methods that use new and old words.  Each run loads the model,
builds the vocabularies (merged with the switch), initialises and loads the engine and runs one step on the host
route; the runs alternate, twice each, and the better of the two is reported.  The card's name and power limit are
read in the same run and printed with the numbers."""
import json
import os
import pickle
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

JAVA14M = dict(token_vocab=1301137, path_vocab=911418, target_vocab=261246, embed_dim=128, code_dim=384, max_contexts=200,
               max_batch=64, top_k=10)
NEW = dict(tokens=200000, paths=100000, names=50000)
BATCH = 64


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def _shell(engine):
    """A Code2VecModel around `engine` with only what its bundle writer uses."""
    from code2vec_b200.b200_model import Code2VecModel
    m = Code2VecModel.__new__(Code2VecModel)
    m.engine, m.world, m.rank, m._save_format = engine, 1, 0, "tf"
    return m


def _write_files(tmp):
    """model/saved (bundle + dictionaries.bin) and data/ft (.dict.c2v + .train.c2v); returns (load path, data prefix)."""
    from code2vec_b200.engine import EngineDims, PathAttentionEngine
    os.makedirs(os.path.join(tmp, "model"))
    os.makedirs(os.path.join(tmp, "data"))
    T, P, Y = (JAVA14M[k] for k in ("token_vocab", "path_vocab", "target_vocab"))
    with open(os.path.join(tmp, "model", "dictionaries.bin"), "wb") as f:
        for prefix, n in (("t", T - 1), ("m", Y - 1), ("p", P - 1)):     # token, target, path; index 0 is <PAD_OR_OOV>
            words = ["%s%d" % (prefix, i) for i in range(n)]
            pickle.dump({w: i + 1 for i, w in enumerate(words)}, f)
            pickle.dump({i + 1: w for i, w in enumerate(words)}, f)
            pickle.dump(n, f)
    e = PathAttentionEngine(EngineDims(**JAVA14M), device=0, training=True)
    e.init_params()
    e.adam_t = 1234
    load = os.path.join(tmp, "model", "saved")
    _shell(e)._save_inner_model(load)
    e.close()
    hist = {}
    for key, prefix, old, n in (("tok", "t", T - 1, NEW["tokens"]), ("path", "p", P - 1, NEW["paths"]),
                                ("tgt", "m", Y - 1, NEW["names"])):
        h = {"%s%d" % (prefix, i): 5 for i in range(0, old, old // 100)}          # some words the model has
        h.update({"new_%s%d" % (prefix, i): 1 + i % 7 for i in range(n)})
        hist[key] = h
    data = os.path.join(tmp, "data", "ft")
    with open(data + ".dict.c2v", "wb") as f:
        for key in ("tok", "path", "tgt"):
            pickle.dump(hist[key], f)
        pickle.dump(BATCH, f)
    lines = []
    for i in range(BATCH):
        name = "new_m%d" % i if i % 2 else "m%d" % i
        ctx = ["%s,%s,%s" % ("new_t%d" % (i * 7 + j) if j % 2 else "t%d" % j, "new_p%d" % j if j % 3 else "p%d" % j,
                             "t%d" % (i + j)) for j in range(50)]
        lines.append(" ".join([name] + ctx + [""] * (JAVA14M["max_contexts"] - len(ctx))))
    with open(data + ".train.c2v", "w") as f:
        f.write("\n".join(lines) + "\n")
    return load, data


def _time_to_first_step(load, data, extend):
    import torch
    from code2vec_b200.b200_model import Code2VecModel
    from code2vec_b200.config import Config
    os.environ["C2V_EXTEND_VOCAB"] = "1" if extend else "0"
    cfg = Config(set_defaults=True)
    cfg.VERBOSE_MODE = 0
    cfg.DL_FRAMEWORK = "b200"
    cfg.MODEL_LOAD_PATH, cfg.TRAIN_DATA_PATH_PREFIX = load, data
    cfg.TRAIN_BATCH_SIZE = cfg.TEST_BATCH_SIZE = BATCH
    cfg.NUM_TRAIN_EPOCHS = 1
    t0 = time.perf_counter()
    m = Code2VecModel(cfg)
    try:
        built = time.perf_counter() - t0
        first = []
        step = m.trainer.step_host

        def timed(*a, **k):
            loss = step(*a, **k)                  # synchronises
            if not first:
                first.append(time.perf_counter() - t0)
            return loss
        m.trainer.step_host = timed
        m.train()
        torch.cuda.synchronize()
        dims = vars(m._engine_dims())
        return built, first[0], {k: dims[k] for k in ("token_vocab", "path_vocab", "target_vocab")}
    finally:
        m.close_session()


def main():
    print(json.dumps(dict(what="card", card=card())), flush=True)
    os.environ["C2V_BATCH_RING"] = "0"                # train() steps through Trainer.step_host, which is timed
    os.environ.pop("WORLD_SIZE", None)
    tmp = tempfile.mkdtemp(prefix="c2v_extend_rate_")
    try:
        load, data = _write_files(tmp)
        best = {}
        for _ in range(2):
            for extend in (False, True):               # alternated, so both see the same page cache and clocks
                built, first, dims = _time_to_first_step(load, data, extend)
                prev = best.get(extend)
                if prev is None or first < prev[1]:
                    best[extend] = (built, first, dims)
        for extend, (built, first, dims) in sorted(best.items()):
            print(json.dumps(dict(what="load and first step", C2V_EXTEND_VOCAB=int(extend), vocab_sizes=dims,
                                  model_built_s=round(built, 2), first_step_done_s=round(first, 2))), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
