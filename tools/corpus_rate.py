#!/usr/bin/env python
"""`--score_names` and `--nearest` (the command line's write_name_scores / write_nearest) on the host route
(C2V_DEVICE_EVAL=0) and on the GPU route (=1), at java14m's model dims with seeded parameters, over eval_rate.py's
synthetic 65,536-line java14m-shaped test file.  Both routes run in one model, alternating, three passes each after a
warm-up of each; the tool checks that they write identical files.  For the device route it also splits a pass into the
evaluation reader alone (read + parse + take), the GPU work on top of it (forward and c2v_name_scores, or forward, the
vectors' gather and c2v_knn_search) and the rest (formatting on the GPU, the copy back and the file writes), and reports
the device and page-locked memory held.  Prints one JSON line with the card's name and power limit.  Writes only to a
temporary directory."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from eval_rate import JAVA14M, _card, _dataset       # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=65536)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--topn", type=int, default=10)
    args = ap.parse_args()
    import torch
    from code2vec_b200 import similarity
    from code2vec_b200.__main__ import write_name_scores, write_nearest
    from code2vec_b200.b200_model import Code2VecModel
    from code2vec_b200.config import Config
    card = _card()
    tmp = tempfile.mkdtemp(prefix="c2v_corpus_rate_")
    try:
        T, P, Y = JAVA14M
        prefix = _dataset(tmp, args.lines, 200, T - 2, P - 2, Y - 1)
        corpus = prefix + ".test.c2v"
        cfg = Config(set_defaults=True)
        cfg.VERBOSE_MODE = 0
        cfg.DL_FRAMEWORK = "b200"
        cfg.TRAIN_DATA_PATH_PREFIX = prefix                  # the vocabularies come from its dictionary; nothing trains
        cfg.MAX_TOKEN_VOCAB_SIZE, cfg.MAX_PATH_VOCAB_SIZE, cfg.MAX_TARGET_VOCAB_SIZE = T, P, Y
        os.environ.setdefault("C2V_SEED", "7")
        os.environ["C2V_DEVICE_EVAL"] = "1"
        model = Code2VecModel(cfg)
        dims = model.engine.dims
        commands = {"score_names": (lambda: write_name_scores(model, corpus), corpus + ".name_scores"),
                    "nearest": (lambda: write_nearest(model, corpus, args.topn), corpus + ".nearest")}
        try:
            def run(cmd: str, device: bool):
                write, path = commands[cmd]
                model._device_eval = device
                torch.cuda.synchronize()
                t0 = time.time()
                write()
                torch.cuda.synchronize()
                s = time.time() - t0
                with open(path, "rb") as f:
                    return s, f.read()

            out = {"what": "--score_names and --nearest: host route (C2V_DEVICE_EVAL=0) vs device route (=1), one model, "
                           "alternating passes, best of %d after a warm-up" % args.passes,
                   "card_and_power_limit": card, "lines": args.lines, "topn": args.topn,
                   "dims": {"tokens": dims.token_vocab, "paths": dims.path_vocab, "targets": dims.target_vocab,
                            "d": dims.embed_dim, "C": dims.max_contexts, "test_batch": cfg.TEST_BATCH_SIZE},
                   "math_eval": model._math_eval}
            rows = None
            for cmd in commands:
                run(cmd, False)
                run(cmd, True)
                times = {False: [], True: []}
                ref = None
                for _ in range(args.passes):
                    for device in (False, True):
                        s, text = run(cmd, device)
                        times[device].append(s)
                        ref = text if ref is None else ref
                        assert text == ref, "%s: the routes wrote different files" % cmd
                rows = ref.count(b"\n")
                stage = model.corpus_text_stage
                out[cmd] = {"rows": rows, "bytes": len(ref), "identical": True,
                            "host_s": [round(s, 3) for s in times[False]], "device_s": [round(s, 3) for s in times[True]],
                            "host_rows_per_s": round(rows / min(times[False])),
                            "device_rows_per_s": round(rows / min(times[True])),
                            "device_text_bytes_held": stage.peak_device_bytes,
                            "pinned_text_bytes_held": stage.peak_host_bytes,
                            "host_wait_for_format_s": round(stage.format_s, 3), "host_write_s": round(stage.write_s, 3),
                            "best_device_s": min(times[True])}

            # the device route's split: the reader alone, then the GPU work on its batches, the rest is text and files
            model._device_eval = True
            e = model.engine
            reader = model._device_corpus_reader(corpus)
            e.set_option("math_mode", model._math_eval)

            def timed(work):
                torch.cuda.synchronize()
                t0 = time.time()
                model._device_corpus_pass(corpus, work) if work else [b.release() for b in reader]
                torch.cuda.synchronize()
                return time.time() - t0

            read_s = min(timed(None) for _ in range(args.passes))
            scores_s = min(timed(lambda b, n, code: e.name_scores(code, b.tensors[4])) for _ in range(args.passes))
            vec = torch.empty((rows, dims.code_dim), dtype=torch.float32, device=e.dev)

            def gather(b, n, code, at=[0]):
                vec[at[0]:at[0] + n].copy_(code)
                at[0] = (at[0] + n) % rows

            def knn():
                t = timed(gather)
                torch.cuda.synchronize()
                t0 = time.time()
                similarity.nearest_rows_device(model._knn(), vec, args.topn, model._math_eval)
                torch.cuda.synchronize()
                return t + time.time() - t0
            nearest_s = min(knn() for _ in range(args.passes))
            for cmd, gpu_s in (("score_names", scores_s), ("nearest", nearest_s)):
                best = out[cmd].pop("best_device_s")
                out[cmd]["device_split_s"] = {"read_parse_take": round(read_s, 3), "gpu_work": round(gpu_s - read_s, 3),
                                              "format_copy_write_and_rest": round(best - gpu_s, 3)}
            out["reader_device_bytes_held"] = reader.device_bytes()
            out["knn_device_bytes_held"] = model._knn().device_bytes()
            out["card_and_power_limit_after"] = _card()
            print(json.dumps(out))
        finally:
            model.close_session()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
