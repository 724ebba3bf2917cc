"""Times preprocess.main on the host route and on the GPU route (C2V_DEVICE_PREPROCESS, DESIGN.md §6g) over a seeded
synthetic raw corpus of java14m's shape, end to end and per phase, and checks that both routes write the same bytes and
leave the rng in the same state.

The corpus: `methods` training methods with bag sizes from a Pareto law (a long tail past 200, capped at 2000), tokens,
paths and targets drawn from Zipf laws over vocabularies far larger than the cut-offs, plus test and val files of a
tenth of the methods each.  Prints one JSON line; --out also writes it to a file.

    python tools/preprocess_rate.py --methods 20000 --out results/preprocess_rate.json
"""
from __future__ import annotations

import argparse
import json
import os
import random
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _lines(rng: np.random.Generator, n: int):
    bags = np.minimum((rng.pareto(1.2, n) + 1) * 20, 2000).astype(np.int64)
    total = int(bags.sum())
    tok = rng.zipf(1.3, 2 * total) % 2_000_000
    pth = rng.zipf(1.2, total) % 1_500_000
    tgt = rng.zipf(1.4, n) % 400_000
    out, k = [], 0
    for i in range(n):
        b = int(bags[i])
        s, p, d = tok[2 * k:2 * k + b], pth[k:k + b], tok[2 * k + b:2 * k + 2 * b]
        k += b
        ctx = " ".join("t%d,p%d,t%d" % (x, y, z) for x, y, z in zip(s.tolist(), p.tolist(), d.tolist()))
        out.append(("m%d|name " % tgt[i]) + ctx)
    return "\n".join(out) + "\n", total


def write_corpus(directory: str, methods: int, seed: int) -> dict:
    """raw.{train,test,val}.txt under directory; returns their sizes and the training contexts."""
    rng = np.random.default_rng(seed)
    stats = {}
    for role, n in (("train", methods), ("test", max(1, methods // 10)), ("val", max(1, methods // 10))):
        text, total = _lines(rng, n)
        path = os.path.join(directory, "raw.%s.txt" % role)
        with open(path, "w") as f:
            f.write(text)
        stats[role + "_bytes"] = os.path.getsize(path)
        if role == "train":
            stats["contexts"] = total
    return stats


def arguments(directory: str):
    d = lambda name: os.path.join(directory, name)
    return ["--train_data", d("raw.train.txt"), "--test_data", d("raw.test.txt"), "--val_data", d("raw.val.txt"),
            "--max_contexts", "200", "--word_vocab_size", "1301136", "--path_vocab_size", "911417",
            "--target_vocab_size", "261245"]


def gpu_name() -> str:
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                     # reported, not fatal: the timing stands without it
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--methods", type=int, default=20000)
    ap.add_argument("--seed", type=int, default=20240921)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from code2vec_b200 import device_preprocess as D
    from code2vec_b200 import preprocess as P
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("preprocess_rate.py needs a GPU")
    with tempfile.TemporaryDirectory() as tmp:
        stats = write_corpus(tmp, a.methods, a.seed)
        argv = arguments(tmp)
        res = {"corpus": stats, "gpu": gpu_name()}
        # warm-up: the library, the CUDA context and the kernels' first launches are set-up, not preprocessing
        D.main(argv + ["--output_name", os.path.join(tmp, "warm")], rng=random.Random(0), log=lambda s: None)
        for route in ("host", "device"):
            rng, logged = random.Random(a.seed), []
            out = os.path.join(tmp, route)
            t0 = time.perf_counter()
            if route == "host":
                P.main(argv + ["--output_name", out], rng=rng, log=logged.append)
            else:
                box = {}
                D.main(argv + ["--output_name", out], rng=rng, log=logged.append, stats=box)
                res["device_phases_s"] = {k: round(v, 3) for k, v in box["phases_s"].items()}
                res["device_memory"] = box["report"]
                res["histogram_table"] = box["table"]
            dt = time.perf_counter() - t0
            res[route + "_s"] = round(dt, 3)
            res[route + "_contexts_per_s"] = round(stats["contexts"] / dt)
            res[route + "_rng"] = hash(rng.getstate())
        same = all(open(os.path.join(tmp, "host." + n), "rb").read() == open(os.path.join(tmp, "device." + n), "rb").read()
                   for n in ("histo.ori.c2v", "histo.path.c2v", "histo.tgt.c2v", "test.c2v", "val.c2v", "train.c2v",
                             "dict.c2v"))
        res["identical"] = bool(same and res["host_rng"] == res["device_rng"])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    if not res["identical"]:
        raise SystemExit("the routes differ")


if __name__ == "__main__":
    main()
