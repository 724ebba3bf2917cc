#!/usr/bin/env python
"""Cost and reproducibility of the engine option "deterministic" at the java14m shape (B = 1024 x 200, keep 0.75, lazy
Adam as Trainer("single") runs it).

Timing: for uniform and Zipfian indices, full and ragged bags, tf32 and 3xTF32, one engine warms up and then alternates
deterministic off / on in the same process; each arm reports the mean device time of a step (CUDA events around
Trainer.step_device) and of its dx_scatter phase (option "profile").  The card name and power limit are read in the same
run.

Reproducibility: the same seeded `--digest-steps` steps run twice on fresh engines with the option on; the SHA-256 over the
losses, the five parameter tensors and both Adam slots (after c2v_sync_tables) must be equal.  One JSON line per result."""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W = dict(token_vocab=1301137, path_vocab=911418, target_vocab=261246, embed_dim=128, code_dim=384, max_contexts=200, batch=1024)
KEEP = 0.75


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        limit = float(out.splitlines()[0])
    except Exception:
        limit = None
    return name, limit


def make_batches(n, zipf, ragged, seed, dev):
    import torch
    rng = np.random.default_rng(seed)
    B, C = W["batch"], W["max_contexts"]
    out = []
    for _ in range(n):
        def idx(vocab):
            if zipf:        # row 0 (PAD / OOV) and a few rows are hot, as in real data
                return np.minimum(rng.zipf(1.1, (B, C)) - 1, vocab - 1)
            return rng.integers(0, vocab, (B, C))
        lengths = np.clip(np.round(rng.normal(0.6 * C, 0.3 * C, B)), 1, C) if ragged else np.full(B, C)
        mask = (np.arange(C)[None, :] < lengths[:, None])
        arrs = [np.where(mask, idx(W["token_vocab"]), 0), np.where(mask, idx(W["path_vocab"]), 0),
                np.where(mask, idx(W["token_vocab"]), 0)]
        t = [torch.from_numpy(a.astype(np.int32)).to(dev) for a in arrs]
        t.append(torch.from_numpy(mask.astype(np.float32)).to(dev))
        t.append(torch.from_numpy(rng.integers(1, W["target_vocab"], B).astype(np.int32)).to(dev))
        out.append(tuple(t))
    return out


def new_trainer(math, deterministic, seed=1):
    from code2vec_b200.engine import EngineDims, PathAttentionEngine
    from code2vec_b200.trainer import Trainer
    eng = PathAttentionEngine(EngineDims(W["token_vocab"], W["path_vocab"], W["target_vocab"], W["embed_dim"], W["code_dim"],
                                         W["max_contexts"], W["batch"], 10), device=0, training=True)
    eng.init_params(seed=seed)
    eng.set_option("math_mode", math)
    return eng, Trainer(eng, keep_prob=KEEP, seed=seed, deterministic=deterministic)


def timed(eng, tr, batches, steps, start):
    import torch
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for i in range(steps):
        tr.step_device(*batches[(start + i) % len(batches)])
    ev1.record()
    ev1.synchronize()
    return ev0.elapsed_time(ev1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="timed steps per arm and repetition")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3, help="off / on alternations per case")
    ap.add_argument("--digest-steps", type=int, default=20)
    ap.add_argument("--cases", default="uniform-full,uniform-ragged,zipf-full,zipf-ragged")
    ap.add_argument("--maths", default="tf32,3xtf32")
    args = ap.parse_args()
    import torch
    from code2vec_b200.engine import MATH_MODES, PARAM_NAMES
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    name, limit = card()
    print(json.dumps({"card": name, "power_limit_w": limit}), flush=True)
    for math in args.maths.split(","):
        for case in args.cases.split(","):
            dist, bags = case.split("-")
            batches = make_batches(4, dist == "zipf", bags == "ragged", 7, dev)
            eng, tr = new_trainer(MATH_MODES[math], False)
            timed(eng, tr, batches, args.warmup, 0)
            res = {0: [], 1: []}
            step = args.warmup
            for _ in range(args.reps):
                for det in (0, 1):
                    eng.set_option("deterministic", det)
                    eng.set_option("profile", 0)
                    ms = timed(eng, tr, batches, args.steps, step)
                    step += args.steps
                    eng.set_option("profile", 1)
                    eng.phase_stats(reset=True)
                    timed(eng, tr, batches, 4, step)
                    step += 4
                    ph = eng.phase_stats(reset=True)
                    sc = ph.get("dx_scatter", (0.0, 1))
                    res[det].append((ms, sc[0] / max(sc[1], 1)))
            eng.set_option("profile", 0)
            out = {"math": math, "case": case, "card": name, "power_limit_w": limit}
            for det, key in ((0, "atomic"), (1, "deterministic")):
                a = np.array(res[det])
                out[key] = {"step_ms": round(float(np.median(a[:, 0])), 3), "dx_scatter_ms": round(float(np.median(a[:, 1])), 3),
                            "step_ms_all": [round(float(x), 3) for x in a[:, 0]]}
            print(json.dumps(out), flush=True)
            eng.close()
            del eng, tr
            torch.cuda.empty_cache()
    # two seeded runs with the option on: SHA-256 of losses, parameters and Adam slots
    digests = []
    for run in range(2):
        batches = make_batches(4, True, True, 11, dev)
        eng, tr = new_trainer(MATH_MODES["tf32"], True, seed=5)
        losses = []
        for i in range(args.digest_steps):
            losses.append(tr.step_device(*batches[i % len(batches)]).clone())
        eng.sync_tables()
        torch.cuda.synchronize()
        h = hashlib.sha256()
        h.update(torch.cat(losses).cpu().numpy().tobytes())
        for tens in (eng.params, eng.adam_m, eng.adam_v):
            for k in PARAM_NAMES:
                h.update(tens[k].detach().cpu().numpy().tobytes())
        digests.append(h.hexdigest())
        eng.close()
        del eng, tr
        torch.cuda.empty_cache()
    print(json.dumps({"digest_steps": args.digest_steps, "math": "tf32", "case": "zipf-ragged", "sha256": digests,
                      "equal": digests[0] == digests[1], "card": name, "power_limit_w": limit}), flush=True)


if __name__ == "__main__":
    main()
