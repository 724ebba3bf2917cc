"""Times the two ways to rank one engine's target rows, on the same code vectors, in one process:
  slab       : c2v_topk -- the logits GEMM writes the [B, Y] fp32 slab, topk_kernel reads it back;
  candidates : c2v_topk_partial + c2v_topk_merge(world = 1), also timed one by one -- the logits GEMM's epilogue
               keeps each (row, partial slot)'s best k in registers and writes only those lists, which
               topk_merge_kernel merges (the row-sharded prediction path of the fully sharded schedule).
Shapes: the single-GPU java14m head (B = 1024, Y = 261,246, D = 384) and one rank's share of it on 8 GPUs (the global
batch of 8 x 1024 examples against a block of 32,656 rows).  tf32 and 3xTF32; k = 10, normalize 0.  The two paths run
alternately, after a warm-up of both, timed with CUDA events; the results must agree bit for bit.  The card's name and
power limit are read in the same run.

    python tools/topk_micro.py [--reps 10] [--rounds 5] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from code2vec_b200.engine import EngineDims, PathAttentionEngine  # noqa: E402

D, K = 384, 10
SHAPES = [("single GPU head", 1024, 261246), ("world-8 rank share", 8192, 32656)]
MATHS = [("tf32", 1), ("3xTF32", 2)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10, help="calls per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="alternating windows per path")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    info = card()
    print("card: %s" % info, flush=True)
    results = {"card": info, "k": K, "rows": []}
    for name, B, Y in SHAPES:
        eng = PathAttentionEngine(EngineDims(101, 101, Y, 128, D, 8, B, K), device=0, training=False)
        eng.init_params(seed=1)
        code = torch.empty((B, D), device=eng.dev).normal_(generator=torch.Generator(device=eng.dev).manual_seed(2))
        i_p = torch.empty((1, B, K), dtype=torch.int32, device=eng.dev)
        v_p = torch.empty((1, B, K), dtype=torch.float32, device=eng.dev)
        i_m, v_m = torch.empty_like(i_p[0]), torch.empty_like(v_p[0])

        def partial():
            eng.topk_partial(code, 0, K, i_p[0], v_p[0])

        def merge():
            eng.topk_merge(i_p, v_p, None, None, 0, B, 0, i_m, v_m)

        def candidates():
            partial()
            merge()

        def slab():
            return eng.topk(code, 0)

        def window(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / args.reps

        for mname, math in MATHS:
            eng.set_option("math_mode", math)
            for _ in range(3):
                want_i, want_v = slab()
                candidates()
            torch.cuda.synchronize()
            same = torch.equal(want_i, i_m) and torch.equal(want_v.view(torch.int32), v_m.view(torch.int32))
            t = {"slab": [], "candidates": [], "partial": [], "merge": []}
            for _ in range(args.rounds):
                for p in t:
                    t[p].append(window({"slab": slab, "candidates": candidates, "partial": partial, "merge": merge}[p]))
            ms = {p: statistics.median(v) for p, v in t.items()}
            row = dict(shape=name, B=B, Y=Y, D=D, math=mname, identical=same, slab_ms=ms["slab"],
                       candidates_ms=ms["candidates"], partial_ms=ms["partial"], merge_ms=ms["merge"],
                       slab_spread=[min(t["slab"]), max(t["slab"])],
                       candidates_spread=[min(t["candidates"]), max(t["candidates"])])
            results["rows"].append(row)
            print("%-20s B=%-5d Y=%-6d %-6s  slab %7.3f ms [%.3f, %.3f]   candidates %7.3f ms [%.3f, %.3f]   "
                  "(partial %.3f + merge %.3f)   ratio %.2f   identical=%s"
                  % (name, B, Y, mname, ms["slab"], *row["slab_spread"], ms["candidates"], *row["candidates_spread"],
                     ms["partial"], ms["merge"], ms["candidates"] / ms["slab"], same), flush=True)
            if not same:
                raise SystemExit("the two paths disagree")
        eng.close()
        del eng, code
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
