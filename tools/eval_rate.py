#!/usr/bin/env python
"""Code2VecModel.evaluate() on the host (C2V_DEVICE_EVAL=0) and on the GPU (=1), at java14m's model dims (1,301,137
tokens, 911,418 paths, 261,246 targets, d = 128, C = 200) with seeded parameters, over a synthetic java14m-shaped test
file (names drawn from the target vocabulary, plus empty fields, which read as the OOV word, and names outside it).
Both routes run in one model, alternating, three passes each after a warm-up of each; the tool checks that they return
equal results and write identical log.txt files.  For the device route it also times its phases, each pass adding one
stage to the last: the evaluation reader alone (read + parse + take), then forward + top-k, then the metric kernel with
its copy-back; host log writing is the rest of evaluate().  Prints one JSON line with the card's name and power limit
and the host's core count.  Writes only to a temporary directory."""
import argparse
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

JAVA14M = (1301137, 911418, 261246)       # token, path and target vocabulary sizes of the java14m model


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def _dataset(tmp, n_lines, C, n_tok, n_path, n_tgt, seed=0):
    """A dictionary of n_tok / n_path / n_tgt words (the vocabularies add their special words) and a test file."""
    prefix = os.path.join(tmp, "java14m_like")
    rng = np.random.default_rng(seed)
    toks = ["tok%d" % i for i in range(n_tok)]
    paths = [str(1000003 * i % 2147483647 - 1073741823) for i in range(n_path)]
    verbs, nouns = ["get", "set", "is", "to", "add", "run", "make"], ["name", "value", "list", "item", "size", "x"]
    alpha = lambda i: "".join(chr(97 + i // 26 ** j % 26) for j in range(4))     # letters only: the names stay legal
    tgts = ["%s|%s%s" % (verbs[i % 7], nouns[i // 7 % 6], alpha(i)) for i in range(n_tgt)]
    with open(prefix + ".test.c2v", "w") as f:
        for _ in range(n_lines):
            k = int(rng.integers(60, C + 1))
            s = rng.integers(0, n_tok, size=(k, 2))
            p = rng.integers(0, n_path, size=k)
            u = rng.random()
            if u < 0.70:
                name = tgts[int(rng.integers(0, n_tgt))]
            elif u < 0.75:
                name = ""                                        # the OOV word
            else:                                                # outside the vocabulary, some normalising to a word in it
                name = "%s|%s" % (verbs[int(rng.integers(0, 7))], nouns[int(rng.integers(0, 6))])
                if rng.random() < 0.3:
                    name = name.replace("|", "").upper()
            f.write(" ".join([name] + ["%s,%s,%s" % (toks[a], paths[b], toks[c]) for (a, c), b in zip(s, p)]
                             + [""] * (C - k)) + "\n")
    os.symlink(prefix + ".test.c2v", prefix + ".train.c2v")     # the model counts its training examples at start-up
    with open(prefix + ".dict.c2v", "wb") as f:
        for words in (toks, paths, tgts):
            pickle.dump({w: 2 for w in words}, f)
        pickle.dump(n_lines, f)
    return prefix


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=65536)
    ap.add_argument("--passes", type=int, default=3)
    args = ap.parse_args()
    import torch
    from code2vec_b200.b200_model import Code2VecModel
    from code2vec_b200.config import Config
    tmp = tempfile.mkdtemp(prefix="c2v_eval_rate_")
    cwd = os.getcwd()
    try:
        os.chdir(tmp)                                       # evaluate() writes log.txt in the working directory
        T, P, Y = JAVA14M
        prefix = _dataset(tmp, args.lines, 200, T - 2, P - 2, Y - 1)
        cfg = Config(set_defaults=True)
        cfg.VERBOSE_MODE = 0
        cfg.DL_FRAMEWORK = "b200"
        cfg.TRAIN_DATA_PATH_PREFIX = prefix                  # the vocabularies come from its dictionary; nothing trains
        cfg.TEST_DATA_PATH = prefix + ".test.c2v"
        cfg.MAX_TOKEN_VOCAB_SIZE, cfg.MAX_PATH_VOCAB_SIZE, cfg.MAX_TARGET_VOCAB_SIZE = T, P, Y
        os.environ.setdefault("C2V_SEED", "7")
        os.environ["C2V_DEVICE_EVAL"] = "0"
        model = Code2VecModel(cfg)
        dims = model.engine.dims
        try:
            def evaluate(device: bool):
                model._device_eval = device
                torch.cuda.synchronize()
                t0 = time.time()
                res = model.evaluate()
                torch.cuda.synchronize()
                return res, time.time() - t0, open("log.txt", "rb").read()

            evaluate(False)
            evaluate(True)                                  # warm-up: page cache, tables, reader buffers
            host_s, dev_s, ref = [], [], None
            for _ in range(args.passes):
                for device, times in ((False, host_s), (True, dev_s)):
                    res, s, log = evaluate(device)
                    times.append(s)
                    if ref is None:
                        ref = (res, log)
                    assert np.array_equal(res.topk_acc, ref[0].topk_acc) and str(res) == str(ref[0]), "results differ"
                    assert (res.subtoken_precision, res.subtoken_recall, res.subtoken_f1) == (
                        ref[0].subtoken_precision, ref[0].subtoken_recall, ref[0].subtoken_f1), "results differ"
                    assert log == ref[1], "log.txt differs"

            # device phases, each pass one stage more
            reader = model._device_eval_reader()
            e = model.engine
            e.set_option("math_mode", model._math_eval)
            phase = {}
            for stage in ("read", "predict", "score"):
                torch.cuda.synchronize()
                t0 = time.time()
                n = 0
                for b in reader:
                    b.wait()
                    n += b.hi - b.lo
                    if stage != "read":
                        code, _ = e.forward(*b.tensors[:4], want_attention=False)
                        ids, _ = e.topk(code, normalize=False)
                        if stage == "score":
                            reader.score(b, ids)
                    b.release()
                torch.cuda.synchronize()
                phase[stage] = time.time() - t0
                rows = n
            best_dev = min(dev_s)
            out = {"what": "evaluate(): host route (C2V_DEVICE_EVAL=0) vs device route (=1), one model, alternating passes",
                   "card_and_power_limit": _card(), "host_cores": os.cpu_count(), "lines": args.lines, "rows": rows,
                   "dims": {"tokens": dims.token_vocab, "paths": dims.path_vocab, "targets": dims.target_vocab,
                            "d": dims.embed_dim, "C": dims.max_contexts, "test_batch": cfg.TEST_BATCH_SIZE,
                            "top_k": cfg.TOP_K_WORDS_CONSIDERED_DURING_PREDICTION},
                   "host_s": [round(s, 3) for s in host_s], "device_s": [round(s, 3) for s in dev_s],
                   "host_rows_per_s": round(rows / min(host_s)), "device_rows_per_s": round(rows / best_dev),
                   "device_phases_s": {"read_parse_take": round(phase["read"], 3),
                                       "forward_topk": round(phase["predict"] - phase["read"], 3),
                                       "metrics_and_copy_back": round(phase["score"] - phase["predict"], 3),
                                       "host_log_writing_and_rest": round(best_dev - phase["score"], 3)},
                   "device_bytes_held": reader.device_bytes(), "results_equal": True, "log_txt_identical": True}
            print(json.dumps(out))
        finally:
            model.close_session()
    finally:
        os.chdir(cwd)
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
