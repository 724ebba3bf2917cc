#!/usr/bin/env python
"""The sampled softmax on the fully sharded schedule (DESIGN.md §6j, "Several GPUs"), one rank's kernels on one H100:
prints one JSON line per (W, S).

For W in {2, 4, 8} and S in {25, 256, 1024} at the java14m shape (Y = 261,246, D = 384, Bl = 1024 examples per rank,
Bt = W * Bl), an engine holding rank 0's block of target rows (the largest block, and the one log-uniform negatives
crowd into) times, with CUDA events around --calls calls each after a warm-up, in --windows windows that alternate
between the four calls (the median and the spread of the windows are printed):
  sampler  c2v_sample_log_uniform_vocab over the global Y (Bl targets)
  pack     c2v_sampled_pack_rows (S negatives, Bt targets)
  step     c2v_sampled_target_step (the head on Bl examples and the partial target gradients)
  fold     c2v_sampled_target_fold (clearing the block, folding W ranks' partials)
and, from one torch.profiler pass of its own, the device time of each kernel c2v_sampled_target_step launches (the head,
the true-row terms, the negative-row sums), and prints the bytes each collective of the step moves per rank (computed
from the shapes, not measured).  The inputs
are random: uniform targets, the sampler's own negatives.  NVLink time and the step time of a real multi-GPU run are not
measured.  The card's name and power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

Y, D, BL = 261246, 384, 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def collective_bytes(W, S, Bl=BL):
    """Bytes per rank each collective of the sampled step carries (payload of one rank's input or output, fp32)."""
    Bt = W * Bl
    return dict(targets_all_gather=4 * Bt, neg_rows_all_reduce=4 * S * D, true_rows_reduce_scatter=4 * Bt * D,
                g_neg_all_gather=4 * W * S * D, g_true_all_gather=4 * Bt * D, loss_all_gather=4 * W)


def timed(fns, calls, windows):
    """{name: (median, min, max) µs per call} over `windows` alternating windows of `calls` calls of each fn."""
    import torch
    for fn in fns.values():
        for _ in range(5):
            fn()
    per = {k: [] for k in fns}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(windows):
        for k, fn in fns.items():
            a.record()
            for _ in range(calls):
                fn()
            b.record()
            torch.cuda.synchronize()
            per[k].append(a.elapsed_time(b) * 1e3 / calls)
    return {k: [round(sorted(v)[len(v) // 2], 2), round(min(v), 2), round(max(v), 2)] for k, v in per.items()}


def kernel_us(fn, calls):
    """Mean device µs per launch of each kernel of fn() (torch.profiler, CUDA activities), by kernel name."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0)
        for name in ("sampled_softmax_rows_fwd", "sampled_true_grad", "sampled_neg_grad", "loss_reduce"):
            if name in ev.key and ev.count:
                out[name] = round(t / ev.count, 2)
    return out


def rank0_rates(W, S_list, calls, windows):
    import torch
    from code2vec_b200.engine import EngineDims, PathAttentionEngine
    from code2vec_b200.trainer import target_row_block
    r0, r1 = target_row_block(Y, 0, W)
    Bt = W * BL
    eng = PathAttentionEngine(EngineDims(8, 8, r1 - r0, 4, D, 1, Bt, 1), device=0, training=True)
    g = torch.Generator(device=eng.dev).manual_seed(W)
    with torch.no_grad():
        eng.params["tgt"].copy_(torch.randn(eng.params["tgt"].shape, device=eng.dev, generator=g) * 0.05)
    dev, f32 = eng.dev, torch.float32
    tgt_all = torch.randint(0, Y, (Bt,), dtype=torch.int32, device=dev, generator=g)
    target = tgt_all[:BL]
    v = torch.randn((BL, D), device=dev, generator=g) * 0.3
    out = []
    for S in S_list:
        sampled, lq_t, lq_s, _ = eng.sample_log_uniform_vocab(target, S, Y, 1, 1)
        sampled, lq_t, lq_s = sampled.clone(), lq_t.clone(), lq_s.clone()
        z = lambda *shape: torch.zeros(shape, dtype=f32, device=dev)
        neg, true_send, g_neg, g_true = z(S, D), z(Bt, D), z(S, D), z(BL, D)
        g_neg_all, g_true_all, dv, loss_part, loss_parts, loss = z(W, S, D), z(Bt, D), z(BL, D), z(1), z(W), z(1)
        true = true_send[:BL]
        step_no = iter(range(2, 10 ** 9))
        step = lambda: eng.sampled_target_step(v, target, sampled, lq_t, lq_s, neg, true, 1.0 / Bt, dv, g_true, g_neg,
                                               loss_part)
        us = timed(dict(
            sampler=lambda: eng.sample_log_uniform_vocab(target, S, Y, 1, next(step_no)),
            pack=lambda: eng.sampled_pack_rows(sampled, tgt_all, r0, neg, true_send),
            step=step,
            fold=lambda: eng.sampled_target_fold(g_true_all, g_neg_all, tgt_all, sampled, r0, loss_parts, loss)),
            calls, windows)
        owned = int(((sampled >= r0) & (sampled < r1)).sum())
        out.append(dict(what="sharded_sampled_rank0", W=W, S=S, Y=Y, D=D, Bl=BL, Bt=Bt, block_rows=r1 - r0,
                        negatives_in_block=owned, us_median_min_max=us,
                        us_sum_of_medians=round(sum(m for m, _, _ in us.values()), 2),
                        step_kernels_us=kernel_us(step, 20), collective_bytes=collective_bytes(W, S)))
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--worlds", default="2,4,8")
    ap.add_argument("--S", default="25,256,1024")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing here can be measured")
    print(json.dumps(dict(card=card())))
    S_list = [int(s) for s in a.S.split(",")]
    for W in (int(w) for w in a.worlds.split(",")):
        for line in rank0_rates(W, S_list, a.calls, a.windows):
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
