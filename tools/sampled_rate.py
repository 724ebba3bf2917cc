#!/usr/bin/env python
"""Sampled-softmax training on one H100 (DESIGN.md §6j): prints one JSON line per measurement.

  * The unique log-uniform sampler alone (c2v_sample_log_uniform) at Y = 261,246 and S in {25, 256, 1024}, B = 1024:
    device time per call (CUDA events around 200 calls) and the draws per step (num_tries) over those calls.
  * The train step at the java14m shape (B = 1024, C = 200, full bags, uniform indices, keep 0.75, lazy Adam as
    Trainer("single") runs it): the full softmax (Trainer.step_device) against Trainer.step_sampled at S in
    {25, 256, 1024}, in tf32 and 3xTF32.  Timed windows of --steps steps alternate between the four after a warm-up of
    each; then one profiled window per case gives the per-phase means of phase_stats.
The card's name and power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

JAVA14M = dict(token_vocab=1301137, path_vocab=911418, target_vocab=261246, embed_dim=128, code_dim=384, max_contexts=200)
B = 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def sampler_rate(S_list, calls=200):
    import torch
    from code2vec_b200.engine import EngineDims, PathAttentionEngine
    Y = JAVA14M["target_vocab"]
    eng = PathAttentionEngine(EngineDims(8, 8, Y, 4, 4, 1, B, 1), device=0, training=False)
    target = torch.randint(0, Y, (B,), dtype=torch.int32, device=eng.dev)
    out = []
    for S in S_list:
        for t in range(20):
            eng.sample_log_uniform(target, S, 1, 10 ** 6 + t)
        tries = torch.empty(calls, dtype=torch.int64, device=eng.dev)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for t in range(calls):
            eng.sample_log_uniform(target, S, 1, t + 1)
        b.record()
        torch.cuda.synchronize()
        for t in range(calls):              # the draws per step, from the same (seed, step) pairs, untimed
            tries[t:t + 1].copy_(eng.sample_log_uniform(target, S, 1, t + 1)[3])
        n = tries.cpu().numpy()
        out.append(dict(what="sampler", Y=Y, S=S, B=B, us_per_call=round(a.elapsed_time(b) * 1e3 / calls, 2),
                        draws_mean=round(float(n.mean()), 1), draws_min=int(n.min()), draws_max=int(n.max())))
    eng.close()
    return out


def step_rate(math, steps, windows, S_list):
    import torch
    from code2vec_b200.engine import EngineDims, PathAttentionEngine
    from code2vec_b200.trainer import Trainer
    from oracle.path_attention_oracle import Dims, synthetic_batch
    d = JAVA14M
    dims = Dims(**d)
    rng = np.random.default_rng(0)
    batches = []
    for i in range(4):
        src, pth, tgt, mask, target = synthetic_batch(dims, B, seed=100 + i)
        mask[:] = 1.0                                   # full bags, uniform indices
        C = d["max_contexts"]
        src[:] = rng.integers(1, d["token_vocab"], (B, C))
        tgt[:] = rng.integers(1, d["token_vocab"], (B, C))
        pth[:] = rng.integers(1, d["path_vocab"], (B, C))
        batches.append((src, pth, tgt, mask, target))
    ed = EngineDims(d["token_vocab"], d["path_vocab"], d["target_vocab"], d["embed_dim"], d["code_dim"], d["max_contexts"], B, 10)
    cases = [("full", 0)] + [("sampled", S) for S in S_list]
    engines = {}
    for kind in ("full", "sampled"):                    # one engine per loss: the sampled one keeps its target rows lazy
        eng = PathAttentionEngine(ed, device=0)
        eng.init_params()
        eng.set_option("math_mode", math)
        tr = Trainer(eng, keep_prob=0.75, seed=5)
        dev = [[eng.to_device(x, torch.int32 if x.dtype != np.float32 else torch.float32) for x in bt] for bt in batches]
        engines[kind] = (eng, tr, dev)

    def run(case, n):
        kind, S = case
        eng, tr, dev = engines[kind]
        for i in range(n):
            bt = dev[i % len(dev)]
            if S:
                tr.step_sampled(*bt, S)
            else:
                tr.step_device(*bt)

    for case in cases:
        run(case, 5)
    torch.cuda.synchronize()
    ms = {case: [] for case in cases}
    for w in range(windows):
        for case in cases:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            run(case, steps)
            b.record()
            b.synchronize()
            ms[case].append(a.elapsed_time(b) / steps)
    out = []
    for case in cases:
        eng = engines[case[0]][0]
        eng.set_option("profile", 1)
        eng.phase_stats(reset=True)
        run(case, steps)
        ph = eng.phase_stats(reset=True)
        eng.set_option("profile", 0)
        per = {k: round(v[0] / steps, 3) for k, v in sorted(ph.items())}
        t = np.array(ms[case])
        out.append(dict(what="train_step", math={1: "tf32", 2: "3xtf32"}[math], loss=case[0], S=case[1],
                        ms_per_step_median=round(float(np.median(t)), 3), ms_per_step_min=round(float(t.min()), 3),
                        ms_per_step_max=round(float(t.max()), 3), windows=windows, steps_per_window=steps,
                        phase_ms_per_step=per))
    for eng, _, _ in engines.values():
        eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    gpu = card()
    rows = [dict(r, card=gpu) for r in sampler_rate([25, 256, 1024])]
    for math in (1, 2):
        rows += [dict(r, card=gpu) for r in step_rate(math, args.steps, args.windows, [25, 256, 1024])]
    for r in rows:
        print(json.dumps(r))
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(json.dumps(r) for r in rows) + "\n")


if __name__ == "__main__":
    main()
