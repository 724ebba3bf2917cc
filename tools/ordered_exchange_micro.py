#!/usr/bin/env python
"""Kernel cost and record count of the two inbox routes of the embedding-gradient exchange on row-sharded tables: the
plain push (one inbox row per context entry, folded with atomics) and option "ordered_exchange" (one sorted, fixed-order
sum per distinct row, folded in rank order).

One process, TWO EMULATED RANKS ON ONE GPU (tests/emulated_ranks.py): java14m shape, B = 1024 x 200 per rank, tf32, keep
0.75, uniform and Zipfian indices, full and ragged bags.  Both "peers" live in the same HBM and the two ranks' kernels
serialise on the one device, so this gives the cost of the kernels and the reduction in pushed records -- not an NVLink
transfer time and not a multi-GPU step time.

Both ranks' engines are set up once with an inbox bound; the option is switched between windows, so the two routes
alternate on the same engines after a warm-up of both.  Per rank and route: the medians over the windows of the mean
`dx_scatter` (the sender's half) and `inbox_apply` (the owner's half) phase times, and the records pushed against the live
entries.  The card's name and power limit are read in the same run.  One JSON line per result.

    python tools/ordered_exchange_micro.py [--steps 4] [--rounds 3] [--warmup 3]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from deterministic_step import KEEP, W, card, make_batches  # noqa: E402
from tests.emulated_ranks import EmulatedGroup, emulate_ipc, run_ranks  # noqa: E402

WORLD = 2


class _Patch:
    """What EmulatedGroup.install needs of pytest's monkeypatch."""

    @staticmethod
    def setattr(obj, name, value, raising=True):
        setattr(obj, name, value)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4, help="profiled steps per window")
    ap.add_argument("--rounds", type=int, default=3, help="alternating windows per route")
    ap.add_argument("--warmup", type=int, default=3, help="steps per route before the first window")
    ap.add_argument("--cases", default="uniform-full,uniform-ragged,zipf-full,zipf-ragged")
    args = ap.parse_args()
    import torch
    from code2vec_b200.engine import MATH_MODES, EngineDims, PathAttentionEngine
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    name, limit = card()
    print(json.dumps({"card": name, "power_limit_w": limit, "emulated_ranks_on_one_gpu": WORLD}), flush=True)
    group = EmulatedGroup(WORLD).install(_Patch)
    engines = []
    for r in range(WORLD):
        e = PathAttentionEngine(EngineDims(W["token_vocab"], W["path_vocab"], W["target_vocab"], W["embed_dim"], W["code_dim"],
                                           W["max_contexts"], W["batch"], 10), device=0, training=True)
        e.init_params(seed=1)
        e.set_option("math_mode", MATH_MODES["tf32"])
        e.set_option("profile", 1)
        engines.append(e)
    emulate_ipc(engines)
    run_ranks(WORLD, lambda r: engines[r].enable_table_sharding(None, push_grads=True), group)
    d = W["embed_dim"]

    def step(batches, t):
        """One exchange on both ranks: backward passes, the barrier a collective would give, folds, gradients cleared."""
        for r, e in enumerate(engines):
            e.train_step(*batches[r], keep=KEEP, seed=1 + r, step=t)
        torch.cuda.synchronize()
        for e in engines:
            e.apply_scatter_inbox()
        for e in engines:
            for n in ("tok", "path"):
                e.shard_grads[n].zero_()
        torch.cuda.synchronize()

    def window(batches, ordered, steps, t):
        for e in engines:
            e.set_option("ordered_exchange", ordered)
            e.phase_stats(reset=True)
        for i in range(steps):
            step(batches, t + i)
        out = []
        for e in engines:
            ph = e.phase_stats(reset=True)
            out.append([ph[k][0] / ph[k][1] for k in ("dx_scatter", "inbox_apply")] + [e.get_option("ordered_exchange_rows")])
        return out

    for case in args.cases.split(","):
        dist, bags = case.split("-")
        batches = make_batches(WORLD, dist == "zipf", bags == "ragged", 7, dev)
        entries = [3 * int(b[3].sum().item()) for b in batches]
        t = 1
        for ordered in (0, 1):
            window(batches, ordered, args.warmup, t)
            t += args.warmup
        res = {0: [], 1: []}
        for _ in range(args.rounds):
            for ordered in (0, 1):
                res[ordered].append(window(batches, ordered, args.steps, t))
                t += args.steps
        for r in range(WORLD):
            out = {"case": case, "rank": r, "live_entries": entries[r], "card": name, "power_limit_w": limit}
            for ordered, key in ((0, "plain_push"), (1, "ordered_exchange")):
                a = np.array([w[r] for w in res[ordered]], dtype=np.float64)
                records = int(a[-1, 2]) if ordered else entries[r]        # plain: a row per live entry (masked ones send an id only)
                out[key] = {"dx_scatter_ms": round(float(np.median(a[:, 0])), 3),
                            "inbox_apply_ms": round(float(np.median(a[:, 1])), 3), "records": records,
                            "pushed_mb": round(records * (d * 4 + 4) / 1e6, 1)}
            print(json.dumps(out), flush=True)
    for e in engines:
        e.set_option("ordered_exchange", 0)
        e.close()


if __name__ == "__main__":
    main()
