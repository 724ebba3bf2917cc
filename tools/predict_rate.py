#!/usr/bin/env python
"""`--predict` on the host (C2V_DEVICE_PREDICT=0: __main__.print_predictions, one method per engine call) and on the GPU
(=1: Code2VecModel.print_predictions_device), at java14m's model dims (1,301,137 tokens, 911,418 paths, 261,246 targets,
d = 128, C = 200) with seeded parameters and the default evaluate/predict arithmetic, over one seeded synthetic
extractor output: names from the target vocabulary, tokens from the token vocabulary, extractor-shaped path strings,
Zipf-sized bags capped at 200.  Both routes run in one model after a warm-up of each on a small input.  Then the
device route is timed --passes times, with a host pass after each of the first --host-passes of them (the host route
takes minutes per pass); every pass must write the same bytes.  Last, the device route is timed --passes times with
--export_code_vectors (the code vectors' text; no host pass).  Prints one JSON line with the times, methods per
second, the memory the device route held, and the card's name and power limit.  Writes only to a temporary
directory."""
import argparse
import io
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

from eval_rate import JAVA14M, _card, _dataset            # noqa: E402
from tests.predict_inputs import synthetic_lines           # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--methods", type=int, default=100000)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--host-passes", type=int, default=1)
    args = ap.parse_args()
    import torch
    from code2vec_b200.__main__ import print_predictions
    from code2vec_b200.b200_model import Code2VecModel
    from code2vec_b200.config import Config
    from code2vec_b200.device_predict import split_source_lines
    tmp = tempfile.mkdtemp(prefix="c2v_predict_rate_")
    try:
        T, P, Y = JAVA14M
        prefix = _dataset(tmp, 16, 200, T - 2, P - 2, Y - 1)      # the dictionaries; its 16 lines are not used
        cfg = Config(set_defaults=True)
        cfg.VERBOSE_MODE = 0
        cfg.DL_FRAMEWORK = "b200"
        cfg.TRAIN_DATA_PATH_PREFIX = prefix
        cfg.MAX_TOKEN_VOCAB_SIZE, cfg.MAX_PATH_VOCAB_SIZE, cfg.MAX_TARGET_VOCAB_SIZE = T, P, Y
        os.environ.setdefault("C2V_SEED", "7")
        os.environ.pop("C2V_MATH", None)
        model = Code2VecModel(cfg)
        tok = [model.vocabs.token_vocab.index_to_word[i] for i in range(2, 50002)]
        tgt = [model.vocabs.target_vocab.index_to_word[i] for i in range(1, 20001)]

        def data_of(n, seed):
            return ("\n".join(synthetic_lines(n, seed, tok, tgt, max_bag=200, n_paths=5000, zipf=1.3,
                                              specials=False)) + "\n").encode("ascii")

        def host(data):
            out = io.BytesIO()
            w = io.TextIOWrapper(out, encoding="utf-8", newline="\n", write_through=True)
            torch.cuda.synchronize()
            t0 = time.time()
            print_predictions(cfg, model, split_source_lines(data, True), out=w)
            torch.cuda.synchronize()
            return time.time() - t0, out.getvalue()

        def device(data, export=False):
            out = io.BytesIO()
            cfg.EXPORT_CODE_VECTORS = export
            torch.cuda.synchronize()
            t0 = time.time()
            assert model.print_predictions_device(data, True, out)
            cfg.EXPORT_CODE_VECTORS = False
            torch.cuda.synchronize()
            return time.time() - t0, out.getvalue()

        try:
            warm = data_of(2000, 1)
            assert host(warm)[1] == device(warm)[1], "warm-up outputs differ"
            data = data_of(args.methods, 2)
            host_s, dev_s, ref = [], [], None
            for i in range(args.passes):
                ds, db = device(data)
                dev_s.append(ds)
                ref = db if ref is None else ref
                assert db == ref, "device passes differ"
                if i < args.host_passes:
                    hs, hb = host(data)
                    host_s.append(hs)
                    assert hb == ref, "outputs differ"
            export_s = []
            for _ in range(args.passes):
                es, eb = device(data, export=True)
                export_s.append(es)
            methods = ref.count(b"Original name:\t")
            p = model._dev_predictor
            bags = [len([f for f in line.split(b" ")[1:] if f]) for line in data.split(b"\n")]
            out = {"what": "--predict: host route (C2V_DEVICE_PREDICT=0) vs device route (=1), one model, alternating",
                   "card_and_power_limit": _card(), "host_cores": os.cpu_count(), "methods": methods,
                   "input_mb": round(len(data) / 1e6, 1), "output_mb": round(len(ref) / 1e6, 1),
                   "output_mb_with_code_vectors": round(len(eb) / 1e6, 1),
                   "mean_bag": round(float(np.mean(bags)), 1),
                   "math": {0: "fp32", 1: "tf32", 2: "3xtf32"}[model._math_eval],
                   "dims": {"tokens": model.engine.dims.token_vocab, "paths": model.engine.dims.path_vocab,
                            "targets": model.engine.dims.target_vocab, "C": cfg.MAX_CONTEXTS,
                            "test_batch": cfg.TEST_BATCH_SIZE},
                   "host_s": [round(s, 2) for s in host_s], "device_s": [round(s, 3) for s in dev_s],
                   "device_with_code_vectors_s": [round(s, 3) for s in export_s],
                   "host_methods_per_s": round(methods / min(host_s)), "device_methods_per_s": round(methods / min(dev_s)),
                   "device_bytes_held": p.device_bytes() + p.vocabs.nbytes(), "pinned_bytes": p.pinned_bytes,
                   "outputs_identical": True}
            print(json.dumps(out))
        finally:
            model.close_session()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
