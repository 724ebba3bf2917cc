"""Rate of the nearest-neighbour search (csrc/knn.cu, DESIGN.md §6h) on seeded tables of the java14m shape, in each math
mode, against torch.mm + torch.topk in fp32 with tf32 off on the same card:
  (a) one most_similar query against the target table (261,245 x 384) and the token table (1,301,136 x 128);
  (b) the 10 nearest names of every target name (nq = 261,245), start to finish: TFLOP/s over 2 nq N d, the device
      time split into the GEMM (with its candidate epilogue) and the selection (merge, exclusion);
  (c) all-pairs nearest methods over 200,000 synthetic code vectors (d = 384).
Every result is checked: each returned similarity of a sample of queries within tests/similarity_model.value_bound of
the float64 score of the same row.  Prints the card's name and power limit, then one JSON line per measurement.

    python tools/similar_rate.py [--out results.json] [--quick]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODES = {0: "fp32", 1: "tf32", 2: "3xtf32"}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out.splitlines()[0] if out else "unknown"


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e3, out


def torch_route(table, q, k, exclude_self_rows=None, chunk=2048):
    """fp32 torch.mm + torch.topk of the scores (T . q) / |T|, k + 1 taken and the own row dropped when asked."""
    import torch
    inv = 1.0 / torch.linalg.vector_norm(table, dim=1)
    ids, vals = [], []
    for s in range(0, q.shape[0], chunk):
        sc = torch.mm(q[s:s + chunk], table.T) * inv
        sc = torch.nan_to_num(sc, nan=-float("inf"))
        v, i = torch.topk(sc, k + (1 if exclude_self_rows is not None else 0), dim=1)
        ids.append(i)
        vals.append(v)
    return torch.cat(ids), torch.cat(vals)


def check(idx, val, table, q, bound, rows=256):
    """Each returned similarity within `bound` of the fp64 score of the same row (a sample of queries)."""
    import torch
    pick = torch.linspace(0, q.shape[0] - 1, min(rows, q.shape[0]), device=q.device).long()
    t64 = table.double()
    s = (q[pick].double() @ t64.T) / torch.linalg.vector_norm(t64, dim=1)
    got = idx[pick].long().clamp(max=table.shape[0] - 1)
    exact = torch.gather(s, 1, got)
    ok = idx[pick] != np.iinfo(np.int32).max
    err = float(((val[pick].double() - exact).abs() * ok).max())
    assert err <= bound, (err, bound)
    return err


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="smaller (b) and (c) for a rehearsal")
    args = ap.parse_args()
    import torch
    from code2vec_b200.similarity import NearestNeighbours, nearest_rows
    from tests.similarity_model import value_bound
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    info = card()
    print("card: %s (name, power limit, max SM clock)" % info, flush=True)
    results = []

    def emit(rec):
        rec["card"] = info
        results.append(rec)
        print(json.dumps(rec), flush=True)

    g = torch.Generator(device=dev).manual_seed(2024)
    tables = {"target": torch.randn((261245, 384), generator=g, device=dev),
              "token": torch.randn((1301136, 128), generator=g, device=dev)}
    nn = NearestNeighbours(dev)
    # (a) one query
    for name, t in tables.items():
        q = t[7:8] / torch.linalg.vector_norm(t[7])
        ms_t, _ = timed(lambda: torch_route(t, q, 10), 20)
        for mode in MODES:
            nn.bind(t, mode)
            torch.cuda.synchronize()
            ms, (idx, val) = timed(lambda: nn.search(q, 10, exclude=[[7]]), 20)
            err = check(idx, val, t, q, value_bound(mode, t.shape[1]))
            emit({"case": "a", "table": name, "mode": MODES[mode], "ms": round(ms, 4), "torch_fp32_ms": round(ms_t, 4),
                  "max_err": err})
    # (b) every target name's 10 nearest
    t = tables["target"]
    nq = 20000 if args.quick else t.shape[0]
    N, d = t.shape
    for mode in MODES:
        nn.bind(t, mode)
        q = nn.queries(np.arange(nq), np.ones(nq, np.float32), np.arange(nq + 1))
        torch.cuda.synchronize()
        nn.profile(True)
        t0 = time.perf_counter()
        idx, val = nn.search(q, 10, exclude_self=True)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        gemm_ms, sel_ms = nn.profile(False)
        err = check(idx, val, t, q, value_bound(mode, d))
        emit({"case": "b", "mode": MODES[mode], "nq": nq, "N": N, "d": d, "wall_s": round(wall, 3),
              "tflops": round(2.0 * nq * N * d / wall / 1e12, 2), "gemm_ms": round(gemm_ms, 1),
              "select_ms": round(sel_ms, 1), "device_mb": round(nn.device_bytes() / 1e6, 1), "max_err": err})
    qn = t[:nq] / torch.linalg.vector_norm(t[:nq], dim=1, keepdim=True)
    t0 = time.perf_counter()
    torch_route(t, qn, 10, exclude_self_rows=True)
    torch.cuda.synchronize()
    emit({"case": "b", "mode": "torch fp32 mm + topk", "nq": nq, "wall_s": round(time.perf_counter() - t0, 3)})
    del tables
    # (c) all-pairs nearest methods
    n_vec = 20000 if args.quick else 200000
    v = torch.randn((n_vec, 384), generator=g, device=dev)
    for mode in MODES:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        idx, val = nearest_rows(nn, v, 10, mode)
        wall = time.perf_counter() - t0
        qv = v / torch.linalg.vector_norm(v, dim=1, keepdim=True)
        err = check(torch.from_numpy(idx).to(dev), torch.from_numpy(val).to(dev), v, qv, value_bound(mode, 384))
        emit({"case": "c", "mode": MODES[mode], "n": n_vec, "wall_s": round(wall, 3),
              "tflops": round(2.0 * n_vec * n_vec * 384 / wall / 1e12, 2), "max_err": err})
    nn.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
